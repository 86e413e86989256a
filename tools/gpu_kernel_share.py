"""Per-kernel device time of the planning tick (torch.profiler, CUDA activities), GPU box:
    python tools/gpu_kernel_share.py [--lattice l216] [--batch 10000] [--filt-window 5] [--ticks 20] [--stateful]
                                     [--pred-points N] [--objects N]
Prints one JSON line: the card, its power limit, and per kernel the time per tick and the share of all kernel time."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch  # noqa: E402

from bench_objects import with_objects  # noqa: E402
from bench_pred import with_predictions  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from tests import helpers as H  # noqa: E402
from graphbasedlocaltrajectoryplanner_b200.planner import BatchPlanner  # noqa: E402
from graphbasedlocaltrajectoryplanner_b200.scenarios import Track, make_scenarios  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--lattice", default="l216")
ap.add_argument("--batch", type=int, default=10000)
ap.add_argument("--filt-window", type=int, default=1)
ap.add_argument("--ticks", type=int, default=20)
ap.add_argument("--stateful", action="store_true", help="time stateful ticks (next_tick) instead of first ticks")
ap.add_argument("--pred-points", type=int, default=0, help="N-point prediction array on every object (bench_pred.py)")
ap.add_argument("--objects", type=int, default=0, help="objects filled up to N per scenario (bench_objects.py)")
args = ap.parse_args()

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                      text=True).stdout.strip().splitlines()[0]
g = H.golden("ticks_%s.npz" % args.lattice)
track = Track(H.track_csv_for(args.lattice))
sc = with_predictions(with_objects(make_scenarios(track, args.batch, seed=12345, n_obj_min=1, n_obj_max=3), args.objects,
                                   track), args.pred_points)
pl = BatchPlanner(H.lattice_for(args.lattice), online=dict(filt_window_width=args.filt_window), device="cuda:0",
                  stateful=args.stateful)
pl.set_vel_params(ax_max_machines=g["ax_max_machines"], vel_max=100.0, gg_scale=1.0, local_gg=(5.0, 5.0), safety_d=30.0)
pl.stage_scenarios(sc)
pl.upload()
pl.set_startpos()
pl.tick()


def one():
    if args.stateful:   # execute an action the last tick returned (the largest action id present)
        sel = pl.t["action_id"].max(dim=0).values.clamp(min=0).cpu().numpy()
        pl.next_tick(sc, sel_action=sel, t_const=0.05)
    else:
        pl.set_startpos()
        pl.tick()


for _ in range(5):
    one()
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(args.ticks):
        one()
    torch.cuda.synchronize()
per = {}
for ev in prof.key_averages():
    if ev.device_type == torch.autograd.DeviceType.CUDA and not ev.key.startswith("Memcpy") \
            and not ev.key.startswith("Memset"):
        name = ev.key.split("(")[0].split("<")[0].replace("void ", "")
        per[name] = per.get(name, 0.0) + ev.device_time_total / 1e3 / args.ticks   # ms per tick
total = sum(per.values())
print(json.dumps({"card": card, "lattice": args.lattice, "batch": args.batch, "filt_window": args.filt_window,
                  "stateful": args.stateful, "pred_points": args.pred_points, "objects": args.objects,
                  "kernel_ms_per_tick": round(total, 4),
                  "kernels": {k: {"ms_per_tick": round(v, 4), "share": round(v / total, 4)}
                              for k, v in sorted(per.items(), key=lambda kv: -kv[1])}}))
