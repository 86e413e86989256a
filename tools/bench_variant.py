"""bench.py's measurement (one GPU) on a changed workload; every other setting and the whole measurement exactly as
bench.py runs them.  Any combination of:
  --objects N       every scenario keeps its objects and gets more, up to N per scenario (workload.with_objects;
                    N at most the batch's own object count is bench.py's batch)
  --pred-points N   every object carries an N-point constant-velocity prediction array (workload.with_predictions;
                    N = 0 is bench.py's batch), applied after --objects
  --filt-window W   the shipped online ini with [SMOOTHING] filt_window_width = W (odd, >= 1)
The JSON line's config block names each given option (objects, pred_points, filt_window_width).

    python tools/bench_variant.py --objects 64 [bench.py arguments, e.g. --steps 20 --warmup 5 --no-cpu-baseline]
"""
import argparse
import contextlib
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    ap = argparse.ArgumentParser(add_help=False)
    ap.add_argument("--objects", type=int)
    ap.add_argument("--pred-points", type=int)
    ap.add_argument("--filt-window", type=int)
    args, rest = ap.parse_known_args()
    if args.objects is not None and args.objects < 1:
        sys.exit("--objects must be >= 1")
    if args.pred_points is not None and args.pred_points < 0:
        sys.exit("--pred-points must be >= 0")
    if args.filt_window is not None and (args.filt_window < 1 or args.filt_window % 2 == 0):
        sys.exit("--filt-window must be a positive odd integer")
    if any(a.startswith("--gpus") and a != "--gpus" for a in rest) or \
            ("--gpus" in rest and rest[rest.index("--gpus") + 1] != "1"):
        sys.exit("tools/bench_variant.py measures one GPU")
    if "--impl" in rest and rest[rest.index("--impl") + 1] != "b200":
        sys.exit("tools/bench_variant.py measures the device path (--impl b200)")

    sys.path.insert(0, REPO)
    import bench
    from graphbasedlocaltrajectoryplanner_b200.scenarios import Track
    from tools import workload
    track = Track(bench.TRACK_CSV)
    make_batch, emit = bench.make_batch, bench.emit
    added = {k: v for k, v in (("objects", args.objects), ("pred_points", args.pred_points),
                                ("filt_window_width", args.filt_window)) if v is not None}

    def make_variant_batch(tag, batch, seed=bench.SEED):
        sc = make_batch(tag, batch, seed=seed)
        if args.objects is not None:
            sc = workload.with_objects(sc, args.objects, track)
        if args.pred_points is not None:
            sc = workload.with_predictions(sc, args.pred_points)
        return sc

    def emit_with_config(line):
        line.setdefault("config", {}).update(added)
        emit(line)
    bench.make_batch, bench.emit = make_variant_batch, emit_with_config
    sys.argv = [os.path.join(REPO, "bench.py")] + rest
    with contextlib.ExitStack() as stack:
        if args.filt_window is not None:
            bench.ONLINE_INI = stack.enter_context(workload.online_ini_with_window(bench.ONLINE_INI, args.filt_window))
        bench.main()


if __name__ == "__main__":
    main()
