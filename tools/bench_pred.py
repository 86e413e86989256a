"""bench.py's measurement with explicit prediction arrays: every object of the benchmark batch carries an N-point
constant-velocity 'prediction' array at 0.1 s spacing (N obstacle discs more per object, OLI:117-119, GLNT:169-189);
every other setting and the whole measurement exactly as bench.py runs them (one GPU).  N = 0 is bench.py's batch
(built-in 0.2 s point).  The JSON line's config block names N.

    python tools/bench_pred.py --pred-points 50 [bench.py arguments, e.g. --steps 20 --warmup 5 --no-cpu-baseline]
"""
import argparse
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DT = 0.1


def with_predictions(sc, n):
    """the batch with an n-point constant-velocity prediction on every object (n = 0: unchanged)."""
    if n == 0:
        return sc
    k = sc.obj.shape[1]
    t = DT * np.arange(1, n + 1)
    x, y, th, v = (sc.obj[:, :, i][..., None] for i in range(4))
    sc.pred = np.stack((x - np.sin(th) * v * t, y + np.cos(th) * v * t), axis=-1)
    sc.n_pred = np.where(np.arange(k)[None, :] < sc.n_obj[:, None], n, -1).astype(np.int32)
    return sc


def main():
    ap = argparse.ArgumentParser(add_help=False)
    ap.add_argument("--pred-points", type=int, required=True)
    args, rest = ap.parse_known_args()
    if args.pred_points < 0:
        sys.exit("--pred-points must be >= 0")
    if any(a.startswith("--gpus") and a != "--gpus" for a in rest) or \
            ("--gpus" in rest and rest[rest.index("--gpus") + 1] != "1"):
        sys.exit("tools/bench_pred.py measures one GPU")
    if "--impl" in rest and rest[rest.index("--impl") + 1] != "b200":
        sys.exit("tools/bench_pred.py measures the device path (--impl b200)")
    sys.path.insert(0, REPO)
    import bench
    make_batch, emit = bench.make_batch, bench.emit
    bench.make_batch = lambda tag, batch, seed=bench.SEED: with_predictions(make_batch(tag, batch, seed=seed),
                                                                             args.pred_points)

    def emit_with_points(line):
        line.setdefault("config", {})["pred_points"] = args.pred_points
        emit(line)
    bench.emit = emit_with_points
    sys.argv = [os.path.join(REPO, "bench.py")] + rest
    bench.main()


if __name__ == "__main__":
    main()
