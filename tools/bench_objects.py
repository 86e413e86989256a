"""bench.py's measurement with long object lists: every scenario of the benchmark batch keeps its objects and gets more,
up to N per scenario (OLI:96-141); every other setting and the whole measurement exactly as bench.py runs them (one
GPU).  The added objects stand 20-500 m ahead of the ego vehicle, every second one 3-15 m beyond the track bounds (an
off-track entry the object filter drops on the device), the others on the track.  N at most the batch's own object
count is bench.py's batch.  The JSON line's config block names N.

    python tools/bench_objects.py --objects 64 [bench.py arguments, e.g. --steps 20 --warmup 5 --no-cpu-baseline]
"""
import argparse
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED = 4242


def with_objects(sc, n, track):
    """the batch with its objects filled up to n per scenario (a fixed seed: the same objects on every call)."""
    k0 = sc.obj.shape[1]
    if n <= k0:
        return sc
    rng = np.random.default_rng(SEED)
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


def main():
    ap = argparse.ArgumentParser(add_help=False)
    ap.add_argument("--objects", type=int, required=True)
    args, rest = ap.parse_known_args()
    if args.objects < 1:
        sys.exit("--objects must be >= 1")
    if any(a.startswith("--gpus") and a != "--gpus" for a in rest) or \
            ("--gpus" in rest and rest[rest.index("--gpus") + 1] != "1"):
        sys.exit("tools/bench_objects.py measures one GPU")
    if "--impl" in rest and rest[rest.index("--impl") + 1] != "b200":
        sys.exit("tools/bench_objects.py measures the device path (--impl b200)")
    sys.path.insert(0, REPO)
    import bench
    from graphbasedlocaltrajectoryplanner_b200.scenarios import Track
    track = Track(bench.TRACK_CSV)
    make_batch, emit = bench.make_batch, bench.emit
    bench.make_batch = lambda tag, batch, seed=bench.SEED: with_objects(make_batch(tag, batch, seed=seed), args.objects,
                                                                         track)

    def emit_with_objects(line):
        line.setdefault("config", {})["objects"] = args.objects
        emit(line)
    bench.emit = emit_with_objects
    sys.argv = [os.path.join(REPO, "bench.py")] + rest
    bench.main()


if __name__ == "__main__":
    main()
