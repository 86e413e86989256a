"""Positions on polylines (ltpl_path_coord_batch) for 100 000 queries:
  s_rows          get_s_coord on per-query 115-row trajectories in the selection layout ([B][115][7] float64, the x / y
                  columns read in place), s_array None (chord sums)
  s_rows_sarr     the same with s_array = the rows' s column, read in place (element stride 7)
  s_raceline      get_s_coord(closed=True) on the shared Monteblanco race line
  inside_bounds   check_inside_bounds on the shared track bounds
Device-event time of one call (tools/workload.timed_ms: L2 flushed before it), after two warm-up calls; the rounds
alternate the variants, each reports the median and the spread over rounds.  Prints one JSON line with the card and its
power limit; it asserts that no variant allocates device memory.

    python tools/bench_path_coord.py [--queries 100000] [--rounds 7]
"""
import argparse
import json
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from graphbasedlocaltrajectoryplanner_b200 import pathcoord as P  # noqa: E402
from tests import helpers as H  # noqa: E402
from tools.workload import card, timed_ms  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queries", type=int, default=100000)
    ap.add_argument("--rounds", type=int, default=7)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    n = a.queries
    rng = np.random.default_rng(1)
    lat = H.lattice_for("default")
    rl = np.asarray(lat.glob_rl, dtype=np.float64)[:-1, 1:3]   # the closed race line, first point once
    b1 = lat.refline + lat.normvec * np.expand_dims(lat.w_right, 1)   # OTH:207-210
    b2 = lat.refline - lat.normvec * np.expand_dims(lat.w_left, 1)
    # trajectories of 115 rows along the race line from random starts, in the selection layout
    start = rng.integers(0, rl.shape[0], size=n)
    k = (start[:, None] + np.arange(115)[None, :]) % rl.shape[0]
    rows = np.zeros((n, 115, 7))
    rows[:, :, 1:3] = rl[k] + rng.normal(0.0, 0.5, size=(n, 1, 2))
    rows[:, 1:, 0] = np.cumsum(np.hypot(*np.moveaxis(np.diff(rows[:, :, 1:3], axis=1), -1, 0)), axis=1)
    sel = torch.as_tensor(rows, device=dev)
    line, s_arr = sel[:, :, 1:3], sel[:, :, 0]
    pos_rows = torch.as_tensor(rows[:, 57, 1:3] + rng.normal(0.0, 2.0, size=(n, 2)), device=dev)
    pos_track = torch.as_tensor(rl[rng.integers(0, rl.shape[0], size=n)] + rng.normal(0.0, 3.0, size=(n, 2)),
                                device=dev)
    d_rl, d_b1, d_b2 = (torch.as_tensor(x, device=dev) for x in (rl, b1, b2))
    s_out = (torch.empty(n, dtype=torch.float64, device=dev), torch.empty((n, 2), dtype=torch.int32, device=dev))
    i_out = torch.empty(n, dtype=torch.int8, device=dev)
    variants = {
        "s_rows": lambda: P.get_s_coord(line, pos_rows, out=s_out),
        "s_rows_sarr": lambda: P.get_s_coord(line, pos_rows, s_array=s_arr, out=s_out),
        "s_raceline": lambda: P.get_s_coord(d_rl, pos_track, closed=True, out=s_out),
        "inside_bounds": lambda: P.check_inside_bounds(d_b1, d_b2, pos_track, out=i_out),
    }
    alloc = {}
    for k, fn in variants.items():
        fn()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        m0 = torch.cuda.memory_allocated()
        fn()
        alloc[k] = torch.cuda.max_memory_allocated() - m0   # 0: every input read in place, out= used
    assert not any(alloc.values()), alloc
    times = {k: [] for k in variants}
    for _ in range(a.rounds):
        for k, fn in variants.items():
            times[k].append(timed_ms(fn))
    res = {k: dict(median_ms=float(np.median(v)), min_ms=float(np.min(v)), max_ms=float(np.max(v)))
           for k, v in times.items()}
    print(json.dumps(dict(card=card(), queries=n, race_line_points=int(rl.shape[0]), bound_points=int(b1.shape[0]),
                          inside=int((i_out == 1).sum()), results=res)))


if __name__ == "__main__":
    main()
