"""
TickGraph -- a first or stateful tick of BatchPlanner captured into CUDA graphs and replayed with no per-tick host work
(DESIGN.md section 11).  Created by BatchPlanner.capture_tick / capture_next_tick.  SplitTickGraph -- the same for a
tick split into its two halves (capture_split_tick / capture_next_split_tick): the paths half, then the velocity half
with the estimates and friction planes the caller computed on the device in between.

A captured tick keeps the pointers and values it was captured with.  What changes between ticks is handled as follows:
  - the inputs: the graph reads static device tensors it owns (``graph.inputs``, ``paths_inputs`` / ``vel_inputs``);
    the caller writes each tick's values into them in place;
  - the trajectory ids: they come from a device counter (buffers.traj_base, k_traj_base) instead of the per-call
    params.traj_base_id;
  - the ping-pong memory of a stateful tick: one graph (per half) per state of the planner's buffers (two parities, a
    third when the first captured tick is also the first with friction planes); a replay runs the graph of the current
    state and then puts the planner's host side where that tick (half) leaves it, which costs no launch;
  - the executed action (sel_action="selected"): the graph stages the planner's selection buffer, and with ``prefer``
    the tick (its velocity half) ends with select(), so every replay leaves the selection the next replay stages.
"""

from __future__ import annotations

from dataclasses import dataclass, replace

import torch

from .planner import check_gg_planes, check_prefer
from .scenarios import DeviceScenarioBatch

_FIELDS = tuple(name for name, _, _ in DeviceScenarioBatch._SPEC)

# graphs of TickGraphs collected while the current stream was capturing a graph: destroying a graph then would
# invalidate that capture, so they are released at the next capture, close() or collection outside one
_DEFERRED = []


def _release_deferred() -> None:
    if not torch.cuda.is_current_stream_capturing():
        while _DEFERRED:
            _DEFERRED.pop().reset()


def _static(a):
    """a device tensor the graph owns, with a's shape, dtype and strides (contiguous where a broadcasts a value)"""
    if not isinstance(a, torch.Tensor):
        return a
    if any(st == 0 and n > 1 for st, n in zip(a.stride(), a.shape)):
        return a.clone(memory_format=torch.contiguous_format)
    return torch.empty_strided(a.shape, a.stride(), dtype=a.dtype, device=a.device).copy_(a)


def _copy_in(what: str, pairs) -> None:
    """(name, static tensor or None, given value) triples: every captured tensor is required, with its shape and
    dtype, and nothing else (ValueError before anything is copied); then the copies, on the current stream"""
    for name, dst, src in pairs:
        if (dst is None) != (src is None):
            raise ValueError("%s: %s %s" % (what, name, "was not captured" if dst is None else "is required"))
        if dst is not None and (not isinstance(src, torch.Tensor) or src.shape != dst.shape or src.dtype != dst.dtype):
            raise ValueError("%s: %s must be a tensor %s of %s" % (what, name, tuple(dst.shape), dst.dtype))
    for _, dst, src in pairs:
        if dst is not None:
            dst.copy_(src, non_blocking=True)


@dataclass
class TickInputs:
    """the static device inputs of a TickGraph.  Write each tick's values into them in place before replay() -- with
    copy_() below or with the tensors' own copy_.  ``t_const`` is a tensor [B], or the float the graph was captured
    with (fixed); ``sc.zones`` is the zone list fixed at capture.  ``sel_action`` is the name "selected" when the graph
    stages the planner's selection (nothing to copy)."""
    sc: DeviceScenarioBatch
    sel_action: torch.Tensor = None
    t_const: object = None
    vel_est: torch.Tensor = None
    restart: torch.Tensor = None

    def copy_(self, sc: DeviceScenarioBatch, sel_action=None, t_const=None, vel_est=None, restart=None) -> None:
        """the next tick's values into the static tensors, on the current stream.  Every tensor the graph was captured
        with is required, with its shape and dtype, and nothing else (ValueError before anything is copied).
        ``sc.zones`` is not read."""
        pairs = [("sc." + n, getattr(self.sc, n), getattr(sc, n)) for n in _FIELDS]
        captured_sel = None if isinstance(self.sel_action, str) else self.sel_action
        pairs += [("sel_action", captured_sel, sel_action)]
        pairs += [(n, getattr(self, n), a) for n, a in (("vel_est", vel_est), ("restart", restart))]
        if isinstance(self.t_const, torch.Tensor):
            pairs.append(("t_const", self.t_const, t_const))
        elif t_const is not None and (self.t_const is None or float(t_const) != self.t_const):
            raise ValueError("TickInputs.copy_: t_const %s" % ("was not captured" if self.t_const is None else
                                                               "was captured as the value %r" % self.t_const))
        _copy_in("TickInputs.copy_", pairs)


@dataclass
class VelInputs:
    """the static device inputs of a SplitTickGraph's velocity half: ``pos_est`` [B][2], ``vel_est`` [B] and the
    friction planes ``ax``, ``ay`` [NSLOT][B][P], float64; None where the capture had none.  Write them in place
    between replay_paths() and replay_vel_profile(), with copy_() or with device code of your own."""
    pos_est: torch.Tensor = None
    vel_est: torch.Tensor = None
    ax: torch.Tensor = None
    ay: torch.Tensor = None

    def copy_(self, pos_est=None, vel_est=None, local_gg=None) -> None:
        """the velocity half's values into the static tensors, on the current stream, with the rule of
        TickInputs.copy_: everything captured is required, nothing else is accepted.  ``local_gg`` = (ax, ay)."""
        if local_gg is not None and (not isinstance(local_gg, (tuple, list)) or len(local_gg) != 2):
            raise ValueError("VelInputs.copy_: local_gg must be the pair (ax, ay)")
        ax, ay = (None, None) if local_gg is None else local_gg
        _copy_in("VelInputs.copy_", [("pos_est", self.pos_est, pos_est), ("vel_est", self.vel_est, vel_est),
                                     ("local_gg[0]", self.ax, ax), ("local_gg[1]", self.ay, ay)])


class _CapturedTick(object):
    """what TickGraph and SplitTickGraph share: per state of the planner's buffers one (CUDA graph, host state after
    it) for each half of the tick, the staleness checks and the release of the graphs"""

    def __init__(self, planner, stateful: bool, entries: dict, pool, own_planes: bool = False):
        self.planner = planner
        self.stateful = stateful
        self._entries = entries        # planner._tick_key -> ((CUDAGraph, host state after the half), ...)
        self._pool = pool
        self._own_planes = own_planes  # the velocity half sets its planes: set_local_gg_planes does not make it stale
        self._generation = self._planner_generation()

    @property
    def n_graphs(self) -> int:
        return 0 if self._entries is None else sum(len(halves) for halves in self._entries.values())

    def _planner_generation(self) -> int:
        pl = self.planner
        return pl._generation - (pl._plane_bumps if self._own_planes else 0)

    def _check(self, what: str) -> None:
        if self._entries is None:
            raise ValueError("%s: the graph was closed" % what)
        if self._planner_generation() != self._generation:
            raise ValueError("%s: the planner changed since the capture (allocate, set_vel_params, set_gg_map, "
                             "set_local_gg_planes, set_subbatches or grown input buffers); capture anew" % what)

    def _halves(self, what: str) -> tuple:
        """the graphs of the planner's current buffer state (ValueError on a closed or stale graph, or a state no
        graph was captured in)"""
        self._check(what)
        halves = self._entries.get(self.planner._tick_key(self.stateful))
        if halves is None:
            raise ValueError("%s: the planner's buffers are in a state this graph was not captured in (a first-tick "
                             "graph replays until the next stateful tick); capture anew" % what)
        return halves

    def _run(self, half, ends_tick: bool) -> None:
        graph, after = half
        graph.replay()
        pl = self.planner
        pl._set_host_state(after)
        if ends_tick:
            pl._tick_count += 1

    def close(self) -> None:
        """release the graphs and their memory pool, after waiting for the device (a replay may still run).  Call it
        outside any stream capture of your own: the wait is a device synchronisation."""
        self._release(wait=True)

    def _release(self, wait: bool) -> None:
        entries, self._entries, self._pool = self._entries, None, None
        if entries:
            if wait:
                torch.cuda.synchronize(self.planner.device)
            _DEFERRED.extend(graph for halves in entries.values() for graph, _ in halves)
        _release_deferred()

    def __del__(self):
        # no synchronisation, and no graph destroyed during a capture: the garbage collector may run this while the
        # caller captures a graph of its own.  CUDA frees an executable graph still in flight when its launch completes.
        try:
            self._release(wait=False)
        except Exception:
            pass


class TickGraph(_CapturedTick):
    """A tick captured into CUDA graphs (BatchPlanner.capture_tick / capture_next_tick).  ``inputs`` (TickInputs) are
    the static device inputs; ``replay()`` enqueues the tick on the current stream.  After a replay the planner's
    results, memory and state are those of the same tick run eagerly.  The graph goes stale when the planner changes
    in a way it cannot follow (allocate, set_vel_params, set_gg_map, set_local_gg_planes, set_subbatches, grown input
    buffers): replay() then raises ValueError; capture a new graph.  ``close()`` releases the graphs."""

    def __init__(self, planner, stateful: bool, inputs: TickInputs, entries: dict, pool, prefer=None):
        super().__init__(planner, stateful, entries, pool)
        self.inputs = inputs
        self.prefer = prefer   # the device preference the graph's select() reads (None: no select)

    def replay(self) -> None:
        """one tick from the current graph inputs, on the current stream: a graph launch plus the host side of the tick
        (pointer swaps, tick count); no host synchronisation, no host memory read by the device, no library call.
        Refused with ValueError, changing nothing, on a closed or stale graph, or when the planner's buffers are in a
        state no graph was captured in."""
        (half,) = self._halves("TickGraph.replay")
        self.planner._split_pending = None
        self._run(half, ends_tick=True)


class SplitTickGraph(_CapturedTick):
    """A tick captured as its two halves (BatchPlanner.capture_split_tick / capture_next_split_tick).  ``paths_inputs``
    (TickInputs) feed the paths half, ``vel_inputs`` (VelInputs) the velocity half.  ``replay_paths()`` enqueues the
    paths half; the caller may then read device_results()["path"] and write ``vel_inputs`` with device code of its
    own; ``replay_vel_profile()`` enqueues the velocity half.  Results, memory and ids are those of the same split
    calls run eagerly.  The velocity half is refused unless the planner's last call was this graph's replay_paths(),
    and a replay_paths() is refused while one waits for its velocity half.  Staleness and close() as TickGraph; a
    graph with friction planes sets them itself, so set_local_gg_planes does not make it stale."""

    def __init__(self, planner, stateful: bool, paths_inputs: TickInputs, vel_inputs: VelInputs, entries: dict, pool,
                 prefer=None):
        super().__init__(planner, stateful, entries, pool, own_planes=vel_inputs.ax is not None)
        self.paths_inputs = paths_inputs
        self.vel_inputs = vel_inputs
        self.prefer = prefer   # the device preference the velocity half's select() reads (None: no select)

    def replay_paths(self) -> None:
        """the paths half from ``paths_inputs``, on the current stream, with no host work.  Refused with ValueError,
        changing nothing, like TickGraph.replay, and while an earlier replay_paths() waits for its velocity half."""
        what = "SplitTickGraph.replay_paths"
        if self.planner._split_pending is not None:
            raise ValueError("%s: the last replay_paths() has not had its velocity half (replay_vel_profile())" % what)
        paths, vel = self._halves(what)
        self._run(paths, ends_tick=False)
        self.planner._split_pending = (self, vel)

    def replay_vel_profile(self) -> None:
        """the velocity half from ``vel_inputs``, on the current stream, with no host work.  Refused with ValueError,
        changing nothing, unless the planner's last call was this graph's replay_paths(), and on a closed or stale
        graph."""
        what = "SplitTickGraph.replay_vel_profile"
        pending = self.planner._split_pending
        if pending is None or pending[0] is not self:
            raise ValueError("%s: the planner's last call was not this graph's replay_paths()" % what)
        self._check(what)
        self.planner._split_pending = None
        self._run(pending[1], ends_tick=True)


def _tick_inputs(pl, what: str, stateful: bool, sc, vel_est, sel_action, t_const, restart) -> TickInputs:
    """the refusals of every capture, then the static inputs of the tick's staging (sel_action="selected" stays the
    name: the graph stages the planner's selection buffer)"""
    if not isinstance(sc, DeviceScenarioBatch):
        raise ValueError("%s: needs a DeviceScenarioBatch (a host ScenarioBatch is copied on the host every tick)" % what)
    if pl._gg_map is None and pl._tick.gg and pl._tick.gg_uploaded:
        raise ValueError("%s: uploaded local_gg planes (set_local_gg_planes) are per-tick host data; a friction map "
                         "(set_gg_map) is evaluated inside the tick" % what)
    if stateful:
        if not pl._tick.ticked:
            raise ValueError("%s: no previous tick in this session (capture_tick or tick first)" % what)
        if sc.size != pl.dims.batch:
            raise ValueError("%s: batch of %d scenarios, the session has %d" % (what, sc.size, pl.dims.batch))
        if sel_action is None or t_const is None:
            raise ValueError("%s: sel_action and t_const are required" % what)
    selected = isinstance(sel_action, str)
    if selected:
        pl._selected(sel_action)
    vel_est, sel_action, t_const, restart = pl._device_args(sc, vel_est, None if selected else sel_action, t_const,
                                                            restart)
    return TickInputs(replace(sc, **{n: _static(getattr(sc, n)) for n in _FIELDS}),
                      "selected" if selected else _static(sel_action), _static(t_const), _static(vel_est),
                      _static(restart))


def _check_selected(what: str, sel_action, prefer) -> None:
    """a graph that stages the selection (sel_action="selected") has to make the next one itself: with prefer"""
    if isinstance(sel_action, str) and prefer is None:
        raise ValueError('%s: sel_action="selected" needs prefer, so that every replay leaves the selection the next '
                         'one stages' % what)


def _prefer(pl, what: str, prefer, batch: int):
    """the graph's own device copy of a preference (check_prefer), made before the capture"""
    if prefer is None:
        return None
    try:
        ids = check_prefer(prefer, batch, pl.device)
    except ValueError as e:
        raise ValueError("%s: %s" % (what, e)) from None
    if not isinstance(ids, torch.Tensor):
        ids = torch.as_tensor(ids).to(pl.device)
    return _static(ids)


def _capture(pl, what: str, stateful: bool, halves) -> tuple:
    """one CUDA graph per half (callables) per state of the planner's buffers, from the current state until the
    states repeat; the planner's host side, tick count and generation are left as they were found.  Returns the
    entries and the memory pool."""
    _release_deferred()
    pool = torch.cuda.graph_pool_handle()
    side = torch.cuda.Stream(device=pl.device)
    before = (pl._host_state(), pl._tick_count, pl._generation, pl._plane_bumps, pl._split_pending)
    entries = {}
    try:
        key = pl._tick_key(stateful)
        while key not in entries:
            if len(entries) == 3:
                raise RuntimeError("%s: the planner's buffers did not return to a captured state" % what)
            graphs = []
            for run in halves:
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph, pool=pool, stream=side):
                    run()
                graphs.append((graph, pl._host_state()))
            entries[key] = tuple(graphs)
            key = pl._tick_key(stateful)
    finally:
        pl._set_host_state(before[0])
        pl._tick_count, pl._generation, pl._plane_bumps, pl._split_pending = before[1:]
    return entries, pool


def capture(pl, stateful: bool, sc, vel_est=None, sel_action=None, t_const=None, restart=None, prefer=None) -> TickGraph:
    """BatchPlanner.capture_tick (stateful False) / capture_next_tick (True): refusals, static inputs, preparation,
    then one capture per state of the planner's buffers until the states repeat"""
    what = "capture_next_tick" if stateful else "capture_tick"
    _check_selected(what, sel_action, prefer)
    inputs = _tick_inputs(pl, what, stateful, sc, vel_est, sel_action, t_const, restart)
    prefer = _prefer(pl, what, prefer, sc.size)
    pl._prepare_capture(inputs, stateful, select=prefer is not None)

    def run():
        if stateful:
            pl.next_tick(inputs.sc, inputs.sel_action, inputs.t_const, vel_est=inputs.vel_est, restart=inputs.restart)
        else:
            pl.stage_scenarios(inputs.sc, vel_est=inputs.vel_est)
            pl.set_startpos()
            pl.tick()
        if prefer is not None:
            pl._select(prefer, None, 0)

    entries, pool = _capture(pl, what, stateful, [run])
    return TickGraph(pl, stateful, inputs, entries, pool, prefer)


def capture_split(pl, stateful: bool, sc, vel_est=None, pos_est=None, local_gg=None, sel_action=None, t_const=None,
                  restart=None, prefer=None) -> SplitTickGraph:
    """BatchPlanner.capture_split_tick (stateful False) / capture_next_split_tick (True): the refusals of capture()
    and those of the velocity half's inputs, static inputs, preparation, then the halves of every buffer state"""
    what = "capture_next_split_tick" if stateful else "capture_split_tick"
    _check_selected(what, sel_action, prefer)
    if isinstance(sc, DeviceScenarioBatch):
        B = sc.size
        if pos_est is not None and (not isinstance(pos_est, torch.Tensor) or pos_est.device != pl.device
                                    or pos_est.dtype != torch.float64 or tuple(pos_est.shape) != (B, 2)):
            raise ValueError("%s: pos_est must be a float64 tensor [%d][2] on %s" % (what, B, pl.device))
        if local_gg is not None:
            if pl._gg_map is not None:
                raise ValueError("%s: local_gg planes and a friction map (set_gg_map) exclude each other" % what)
            if not isinstance(local_gg, (tuple, list)) or len(local_gg) != 2:
                raise ValueError("%s: local_gg must be the pair (ax, ay)" % what)
            check_gg_planes(local_gg[0], local_gg[1], B, pl.cap["p_max"], pl.device)
    inputs = _tick_inputs(pl, what, stateful, sc, None, sel_action, t_const, restart)
    vel_est = pl._device_args(sc, vel_est)[0]
    ax, ay = (None, None) if local_gg is None else local_gg
    vel_inputs = VelInputs(*(_static(a) for a in (pos_est, vel_est, ax, ay)))
    prefer = _prefer(pl, what, prefer, sc.size)
    pl._prepare_capture(inputs, stateful, planes=local_gg is not None, select=prefer is not None)

    def paths():
        if stateful:
            pl.next_calc_paths(inputs.sc, inputs.sel_action, inputs.t_const, restart=inputs.restart)
        else:
            pl.stage_scenarios(inputs.sc)
            pl.set_startpos()
            pl.calc_paths()

    def vel():
        if vel_inputs.ax is not None:
            pl.set_local_gg_planes(vel_inputs.ax, vel_inputs.ay)
        if stateful:
            pl.next_calc_vel_profile(pos_est=vel_inputs.pos_est, vel_est=vel_inputs.vel_est)
        else:
            if vel_inputs.pos_est is not None or vel_inputs.vel_est is not None:
                pl.set_estimates(vel_inputs.pos_est, vel_inputs.vel_est)
            pl.calc_vel_profile()
        if prefer is not None:
            pl._select(prefer, None, 0)

    entries, pool = _capture(pl, what, stateful, [paths, vel])
    return SplitTickGraph(pl, stateful, inputs, vel_inputs, entries, pool, prefer)
