"""
TickGraph -- a first or stateful tick of BatchPlanner captured into CUDA graphs and replayed with no per-tick host work
(DESIGN.md section 11).  Created by BatchPlanner.capture_tick / capture_next_tick.

A captured tick keeps the pointers and values it was captured with.  What changes between ticks is handled as follows:
  - the inputs: the graph reads static device tensors it owns (``graph.inputs``); the caller writes each tick's values
    into them in place;
  - the trajectory ids: they come from a device counter (buffers.traj_base, k_traj_base) instead of the per-call
    params.traj_base_id;
  - the ping-pong memory of a stateful tick: one graph per state of the planner's buffers (two parities, a third when
    the first captured tick is also the first with friction planes); a replay runs the graph of the current state and
    then puts the planner's host side where that tick leaves it, which costs no launch.
"""

from __future__ import annotations

from dataclasses import dataclass, replace

import torch

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


@dataclass
class TickInputs:
    """the static device inputs of a TickGraph.  Write each tick's values into them in place before replay() -- with
    copy_() below or with the tensors' own copy_.  ``t_const`` is a tensor [B], or the float the graph was captured
    with (fixed); ``sc.zones`` is the zone list fixed at capture."""
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
        pairs += [(n, getattr(self, n), a) for n, a in (("sel_action", sel_action), ("vel_est", vel_est),
                                                        ("restart", restart))]
        if isinstance(self.t_const, torch.Tensor):
            pairs.append(("t_const", self.t_const, t_const))
        elif t_const is not None and (self.t_const is None or float(t_const) != self.t_const):
            raise ValueError("TickInputs.copy_: t_const %s" % ("was not captured" if self.t_const is None else
                                                               "was captured as the value %r" % self.t_const))
        for name, dst, src in pairs:
            if (dst is None) != (src is None):
                raise ValueError("TickInputs.copy_: %s %s" % (name, "was not captured" if dst is None else "is required"))
            if dst is not None and (not isinstance(src, torch.Tensor) or src.shape != dst.shape or src.dtype != dst.dtype):
                raise ValueError("TickInputs.copy_: %s must be a tensor %s of %s" % (name, tuple(dst.shape), dst.dtype))
        for _, dst, src in pairs:
            if dst is not None:
                dst.copy_(src, non_blocking=True)


class TickGraph(object):
    """A tick captured into CUDA graphs (BatchPlanner.capture_tick / capture_next_tick).  ``inputs`` (TickInputs) are
    the static device inputs; ``replay()`` enqueues the tick on the current stream.  After a replay the planner's
    results, memory and state are those of the same tick run eagerly.  The graph goes stale when the planner changes
    in a way it cannot follow (allocate, set_vel_params, set_gg_map, set_local_gg_planes, set_subbatches, grown input
    buffers): replay() then raises ValueError; capture a new graph.  ``close()`` releases the graphs."""

    def __init__(self, planner, stateful: bool, inputs: TickInputs, entries: dict, pool, generation: int):
        self.planner = planner
        self.stateful = stateful
        self.inputs = inputs
        self._entries = entries        # planner._tick_key -> (CUDAGraph, host state after the tick)
        self._pool = pool
        self._generation = generation

    @property
    def n_graphs(self) -> int:
        return 0 if self._entries is None else len(self._entries)

    def replay(self) -> None:
        """one tick from the current graph inputs, on the current stream: a graph launch plus the host side of the tick
        (pointer swaps, tick count); no host synchronisation, no host memory read by the device, no library call.
        Refused with ValueError, changing nothing, on a closed or stale graph, or when the planner's buffers are in a
        state no graph was captured in."""
        pl = self.planner
        if self._entries is None:
            raise ValueError("TickGraph.replay: the graph was closed")
        if pl._generation != self._generation:
            raise ValueError("TickGraph.replay: the planner changed since the capture (allocate, set_vel_params, "
                             "set_gg_map, set_local_gg_planes, set_subbatches or grown input buffers); capture anew")
        entry = self._entries.get(pl._tick_key(self.stateful))
        if entry is None:
            raise ValueError("TickGraph.replay: the planner's buffers are in a state this graph was not captured in "
                             "(a first-tick graph replays until the next stateful tick); capture anew")
        graph, after = entry
        graph.replay()
        pl._set_host_state(after)
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
            _DEFERRED.extend(graph for graph, _ in entries.values())
        _release_deferred()

    def __del__(self):
        # no synchronisation, and no graph destroyed during a capture: the garbage collector may run this while the
        # caller captures a graph of its own.  CUDA frees an executable graph still in flight when its launch completes.
        try:
            self._release(wait=False)
        except Exception:
            pass


def capture(pl, stateful: bool, sc, vel_est=None, sel_action=None, t_const=None, restart=None) -> TickGraph:
    """BatchPlanner.capture_tick (stateful False) / capture_next_tick (True): refusals, static inputs, preparation,
    then one capture per state of the planner's buffers until the states repeat; the planner's host side is left as
    it was found"""
    what = "capture_next_tick" if stateful else "capture_tick"
    if not isinstance(sc, DeviceScenarioBatch):
        raise ValueError("%s: needs a DeviceScenarioBatch (a host ScenarioBatch is copied on the host every tick)" % what)
    if pl._gg_map is None and pl.buf is not None and pl.buf.gg is not None:
        raise ValueError("%s: uploaded local_gg planes (set_local_gg_planes) are per-tick host data; a friction map "
                         "(set_gg_map) is evaluated inside the tick" % what)
    if stateful:
        if not pl._tick.ticked:
            raise ValueError("%s: no previous tick in this session (capture_tick or tick first)" % what)
        if sc.size != pl.dims.batch:
            raise ValueError("%s: batch of %d scenarios, the session has %d" % (what, sc.size, pl.dims.batch))
        if sel_action is None or t_const is None:
            raise ValueError("%s: sel_action and t_const are required" % what)
    vel_est, sel_action, t_const, restart = pl._device_args(sc, vel_est, sel_action, t_const, restart)
    inputs = TickInputs(replace(sc, **{n: _static(getattr(sc, n)) for n in _FIELDS}), _static(sel_action),
                        _static(t_const), _static(vel_est), _static(restart))
    pl._prepare_capture(inputs, stateful)

    def run():
        if stateful:
            pl.next_tick(inputs.sc, inputs.sel_action, inputs.t_const, vel_est=inputs.vel_est, restart=inputs.restart)
        else:
            pl.stage_scenarios(inputs.sc, vel_est=inputs.vel_est)
            pl.set_startpos()
            pl.tick()

    _release_deferred()
    pool = torch.cuda.graph_pool_handle()
    side = torch.cuda.Stream(device=pl.device)
    before, tick_count = pl._host_state(), pl._tick_count
    entries = {}
    try:
        key = pl._tick_key(stateful)
        while key not in entries:
            if len(entries) == 3:
                raise RuntimeError("%s: the planner's buffers did not return to a captured state" % what)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, pool=pool, stream=side):
                run()
            entries[key] = (graph, pl._host_state())
            key = pl._tick_key(stateful)
    finally:
        pl._set_host_state(before)
        pl._tick_count = tick_count
    return TickGraph(pl, stateful, inputs, entries, pool, pl._generation)
