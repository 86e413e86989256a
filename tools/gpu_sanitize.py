"""compute-sanitizer target (GPU box): one small tick of every kernel on each lattice + the dense velocity microbench.
Run as  compute-sanitizer --tool memcheck|racecheck|initcheck|synccheck python tools/gpu_sanitize.py"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np
from tests import helpers as H
from graphbasedlocaltrajectoryplanner_b200.planner import BatchPlanner
from graphbasedlocaltrajectoryplanner_b200.scenarios import Track, make_scenarios, make_velocity_microbench
from graphbasedlocaltrajectoryplanner_b200.velprofile import calc_vel_profile_batch

n = int(sys.argv[1]) if len(sys.argv) > 1 else 96
VEL = dict(vel_max=100.0, gg_scale=1.0, local_gg=(5.0, 5.0), safety_d=30.0)
for tag in ("default", "l216"):
    g = H.golden("ticks_%s.npz" % tag)
    sc = make_scenarios(Track(H.TRACK_CSV), n, seed=77, n_obj_min=0, n_obj_max=3)
    pl = BatchPlanner(H.lattice_for(tag), device="cuda:0")
    pl.set_vel_params(ax_max_machines=g["ax_max_machines"], **VEL)
    pl.stage_scenarios(sc); pl.upload(); pl.set_startpos(); pl.tick()
    r = pl.records()
    print(tag, "trajectories:", sum(len(x.get("traj", {})) for x in r))
# velocity smoothing (k_smooth): a first tick and a stateful tick at window 5, emergency trajectory on
g = H.golden("ticks_default.npz")
sc = make_scenarios(Track(H.TRACK_CSV), n, seed=78, n_obj_min=0, n_obj_max=3)
ps = BatchPlanner(H.lattice_for("default"), online=dict(filt_window_width=5), device="cuda:0", stateful=True)
ps.set_vel_params(ax_max_machines=g["ax_max_machines"], incl_emerg_traj=True, **VEL)
ps.stage_scenarios(sc); ps.upload(); ps.set_startpos(); ps.tick()
sel = ps.t["action_id"].max(dim=0).values.clamp(min=0).cpu().numpy()   # an action every scenario's tick returned
ps.next_tick(sc, sel_action=sel, t_const=0.1)
r = ps.records()
print("smoothed stateful tick, trajectories:", sum(len(x.get("traj", {})) for x in r))
# long prediction arrays (k_plan's disc stage in chunks of 32): 3 objects x 40 points = 123 discs per scenario, a first
# tick and a stateful tick
from bench_pred import with_predictions  # noqa: E402
sc = with_predictions(make_scenarios(Track(H.TRACK_CSV), n, seed=79, n_obj_min=3, n_obj_max=3), 40)
pp = BatchPlanner(H.lattice_for("default"), device="cuda:0", stateful=True)
pp.set_vel_params(ax_max_machines=g["ax_max_machines"], **VEL)
pp.stage_scenarios(sc); pp.upload(); pp.set_startpos(); pp.tick()
sel = pp.t["action_id"].max(dim=0).values.clamp(min=0).cpu().numpy()
pp.next_tick(sc, sel_action=sel, t_const=0.1)
r = pp.records()
print("long-prediction stateful tick, trajectories:", sum(len(x.get("traj", {})) for x in r))
# long object lists (k_plan's object stage in chunks of 32, a vehicle record per on-track object): 70 objects per
# scenario, every second added one beyond the track bounds, a first tick and a stateful tick
from bench_objects import with_objects  # noqa: E402
tr = Track(H.TRACK_CSV)
sc = with_objects(make_scenarios(tr, n, seed=80, n_obj_min=1, n_obj_max=3), 70, tr)
po = BatchPlanner(H.lattice_for("default"), device="cuda:0", stateful=True)
po.set_vel_params(ax_max_machines=g["ax_max_machines"], **VEL)
po.stage_scenarios(sc); po.upload(); po.set_startpos(); po.tick()
sel = po.t["action_id"].max(dim=0).values.clamp(min=0).cpu().numpy()
po.next_tick(sc, sel_action=sel, t_const=0.1)
r = po.records()
print("70-object stateful tick, trajectories:", sum(len(x.get("traj", {})) for x in r))
# restarts inside a stateful tick (masked k_startpos in front of k_state): every third scenario, a few of them to a
# pose off the track, emergency trajectory on, then a stateful tick without restarts
sc = make_scenarios(Track(H.TRACK_CSV), n, seed=81, n_obj_min=0, n_obj_max=3)
pr = BatchPlanner(H.lattice_for("default"), device="cuda:0", stateful=True)
pr.set_vel_params(ax_max_machines=g["ax_max_machines"], incl_emerg_traj=True, **VEL)
pr.stage_scenarios(sc); pr.upload(); pr.set_startpos(); pr.tick()
sel = pr.t["action_id"].max(dim=0).values.clamp(min=0).cpu().numpy()
mask = np.arange(n) % 3 == 0
sc2 = make_scenarios(Track(H.TRACK_CSV), n, seed=82, n_obj_min=0, n_obj_max=3)
sc.pos[mask], sc.heading[mask], sc.vel[mask] = sc2.pos[mask], sc2.heading[mask], sc2.vel[mask]
sc.pos[:9:3] += 40.0
pr.next_tick(sc, sel_action=sel, t_const=0.1, restart=mask)
sel = pr.t["action_id"].max(dim=0).values.clamp(min=0).cpu().numpy()
pr.next_tick(sc, sel_action=sel, t_const=0.1)
r = pr.records()
print("stateful tick after restarts, trajectories:", sum(len(x.get("traj", {})) for x in r))
mb =make_velocity_microbench(200, 150, seed=3)
vx, ax = calc_vel_profile_batch(pl, mb["kappa"], mb["el"], mb["v_start"], mb["v_end"])
print("dense vx mean", float(np.mean(vx)))
