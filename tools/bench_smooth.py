"""bench.py's measurement with velocity smoothing: the shipped online ini with [SMOOTHING] filt_window_width = W, every
other setting and the whole measurement exactly as bench.py runs them (one GPU).  The JSON line's config block names the
window.

    python tools/bench_smooth.py --filt-window 5 [bench.py arguments, e.g. --steps 20 --warmup 5 --no-cpu-baseline]
"""
import argparse
import os
import shutil
import sys
import tempfile

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

ap = argparse.ArgumentParser(add_help=False)
ap.add_argument("--filt-window", type=int, required=True)
args, rest = ap.parse_known_args()
if args.filt_window < 1 or args.filt_window % 2 == 0:
    sys.exit("--filt-window must be a positive odd integer")
if any(a.startswith("--gpus") and a != "--gpus" for a in rest) or ("--gpus" in rest and rest[rest.index("--gpus") + 1] != "1"):
    sys.exit("tools/bench_smooth.py measures one GPU")
if "--impl" in rest and rest[rest.index("--impl") + 1] != "b200":
    sys.exit("tools/bench_smooth.py measures the device path (--impl b200)")

import bench  # noqa: E402

tmp = tempfile.mkdtemp(prefix="ltpl_bench_smooth_")
try:
    txt = open(bench.ONLINE_INI).read()
    assert txt.count("filt_window_width=1\n") == 1
    ini = os.path.join(tmp, "ltpl_config_online.ini")
    open(ini, "w").write(txt.replace("filt_window_width=1\n", "filt_window_width=%d\n" % args.filt_window))
    bench.ONLINE_INI = ini
    emit = bench.emit

    def emit_with_window(line):
        line.setdefault("config", {})["filt_window_width"] = args.filt_window
        emit(line)
    bench.emit = emit_with_window
    sys.argv = [os.path.join(REPO, "bench.py")] + rest
    bench.main()
finally:
    shutil.rmtree(tmp, ignore_errors=True)
