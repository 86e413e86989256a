"""debug (GPU box): tick time against the number of scenario windows (ltpl_set_subbatches).
usage: python tools/gpu_subbatch.py [tag ...]"""
import os, sys
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import bench
from graphbasedlocaltrajectoryplanner_b200.planner import BatchPlanner
from tools.workload import timed_ms


for tag in (sys.argv[1:] or ["l216", "default", "l430"]):
    for batch in (10000, 5000, 1250):
        pl = BatchPlanner(bench.get_lattice(tag), device="cuda:0")
        pl.set_vel_params(**bench.vel_kwargs())
        pl.stage_scenarios(bench.make_batch(tag, batch)); pl.upload(); pl.set_startpos()
        row = []
        for n in (1, 2, 3, 4, 5, 6, 8):
            pl.set_subbatches(n)
            for _ in range(3):
                pl.tick()
            row.append("%d: %.4f" % (n, sorted(timed_ms(pl.tick) for _ in range(12))[6]))   # median
        print("%-8s B=%-6d tick ms by windows  %s" % (tag, batch, "  ".join(row)), file=sys.__stdout__, flush=True)
