"""compute-sanitizer target (GPU box): one small tick of every kernel on each lattice + the dense velocity microbench.
Run as  compute-sanitizer --tool memcheck|racecheck|initcheck|synccheck python tools/gpu_sanitize.py"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from tests import helpers as H
from tools.workload import with_objects, with_predictions
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
# a first tick and a stateful tick of each case: velocity smoothing (k_smooth) at window 5 with the emergency trajectory
# on; long prediction arrays (k_plan's disc stage in chunks of 32): 3 objects x 40 points = 123 discs per scenario; long
# object lists (k_plan's object stage in chunks of 32, a vehicle record per on-track object): 70 objects per scenario,
# every second added one beyond the track bounds
g = H.golden("ticks_default.npz")
tr = Track(H.TRACK_CSV)
for name, seed, n_obj, variant, online, emerg in (
        ("smoothed", 78, (0, 3), lambda sc: sc, dict(filt_window_width=5), True),
        ("long-prediction", 79, (3, 3), lambda sc: with_predictions(sc, 40), None, False),
        ("70-object", 80, (1, 3), lambda sc: with_objects(sc, 70, tr), None, False)):
    sc = variant(make_scenarios(tr, n, seed=seed, n_obj_min=n_obj[0], n_obj_max=n_obj[1]))
    ps = BatchPlanner(H.lattice_for("default"), online=online, device="cuda:0", stateful=True)
    ps.set_vel_params(ax_max_machines=g["ax_max_machines"], incl_emerg_traj=emerg, **VEL)
    ps.stage_scenarios(sc); ps.upload(); ps.set_startpos(); ps.tick()
    sel = ps.t["action_id"].max(dim=0).values.clamp(min=0).cpu().numpy()   # an action every scenario's tick returned
    ps.next_tick(sc, sel_action=sel, t_const=0.1)
    r = ps.records()
    print(name + " stateful tick, trajectories:", sum(len(x.get("traj", {})) for x in r))
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
# a friction map over part of the track (k_gg_map in front of the velocity kernels), emergency trajectory on: a first
# tick and a stateful tick (the backup brake reads the last tick's map planes)
from tests import gg_map_ref as M
ax, ay = M.surface_map(3.7, x0=-300.0, y0=-150.0, width=500.0, height=350.0)
pm = BatchPlanner(H.lattice_for("default"), device="cuda:0", stateful=True)
pm.set_vel_params(ax_max_machines=g["ax_max_machines"], incl_emerg_traj=True, **VEL)
pm.set_gg_map(ax, ay, -300.0, -150.0, 3.7)
pm.stage_scenarios(sc); pm.upload(); pm.set_startpos(); pm.tick()
sel = pm.t["action_id"].max(dim=0).values.clamp(min=0).cpu().numpy()
pm.next_tick(sc, sel_action=sel, t_const=0.1)
r = pm.records()
print("friction map stateful tick, trajectories:", sum(len(x.get("traj", {})) for x in r))
# scenario inputs from device tensors (k_stage): a first tick with predictions and zones from a DeviceScenarioBatch, then
# a stateful tick with strided object columns, device sel_action / t_const / vel_est and a restart mask
import torch
sc = with_predictions(make_scenarios(Track(H.TRACK_CSV), n, seed=83, n_obj_min=0, n_obj_max=3), 6)
sc.set_zones([{"z%d" % (b % 3): [[20 + b % 3, 20 + b % 3, 21], [0, 1, 0], None, None]} if b % 2 == 0 else None
              for b in range(n)])
pd = BatchPlanner(H.lattice_for("default"), device="cuda:0", stateful=True)
pd.set_vel_params(ax_max_machines=g["ax_max_machines"], incl_emerg_traj=True, **VEL)
dsc = sc.to_device("cuda:0")
pd.stage_scenarios(dsc); pd.upload(); pd.set_startpos(); pd.tick()
wide = torch.zeros((n, dsc.obj.shape[1], 8), dtype=torch.float64, device="cuda:0")
wide[:, :, 2:7] = dsc.obj
dsc.obj = wide[:, :, 2:]
sel = pd.device_results()["action_id"].max(dim=0).values.clamp(min=0)
pd.next_tick(dsc, sel, torch.full((n,), 0.1, dtype=torch.float64, device="cuda:0"), vel_est=dsc.vel * 0.9,
             restart=torch.arange(n, device="cuda:0") % 5 == 0)
r = pd.records()
print("device inputs stateful tick, trajectories:", sum(len(x.get("traj", {})) for x in r))
# a stateful tick captured into CUDA graphs (one per ping-pong parity, k_traj_base behind the windows) and replayed 4
# times with the next sel_action copied into its inputs
graph = pd.capture_next_tick(dsc, sel, 0.1, vel_est=dsc.vel * 0.9)
for _ in range(4):
    graph.inputs.copy_(dsc, pd.device_results()["action_id"].max(dim=0).values.clamp(min=0), vel_est=dsc.vel * 0.9)
    graph.replay()
graph.close()
r = pd.records()
print("replayed stateful tick, trajectories:", sum(len(x.get("traj", {})) for x in r))
mb = make_velocity_microbench(200, 150, seed=3)
vx, ax = calc_vel_profile_batch(pl, mb["kappa"], mb["el"], mb["v_start"], mb["v_end"])
print("dense vx mean", float(np.mean(vx)))
# follow-mode profiles (k_velfollow): ragged lengths with per-point friction and the race line in shared memory, then
# constant friction with the race line read through L2 (resampled to 4 x its points, above the shared-memory capacity)
from tests import vel_follow_ref as R
from graphbasedlocaltrajectoryplanner_b200.velprofile import VelocityPlanner
rl = R.race_line()
fi = R.random_inputs(70, 90, 5, rl)
fs = np.cumsum(fi["el"], axis=1) - fi["el"]
fgg = np.stack((4.5 + 0.5 * np.sin(fs / 50.0), 5.0 + 0.5 * np.cos(fs / 70.0)), axis=-1)
t4 = np.arange(4 * (rl.shape[0] - 1)) / 4.0
rl4 = np.column_stack([np.interp(t4, np.arange(rl.shape[0]), rl[:, c]) for c in range(5)])
rl4 = np.vstack((rl4, rl4[:1]))
rl4[-1, 0] = rl[-1, 0]
for glob, gg, n_pts in ((rl, fgg, np.random.default_rng(6).integers(2, 91, size=70)), (rl4, (5.0, 5.0), None)):
    fv = VelocityPlanner(device="cuda:0", veh_param_dyn_model_exp=1.5, len_veh=4.7, follow_control_type="PD",
                         follow_control_params={"c_p": 1.25, "k_d": 0.025, "k_p": 0.2}, glob_rl=glob)
    fv.update_dyn_parameters(vel_max=60.0, gg_scale=0.9, ax_max_machines=g["ax_max_machines"])
    fx, _, ftc, fvb = fv.calc_vel_profile_follow(fi["kappa"], fi["el"], gg, fi["v_start"], fi["v_ego"], fi["v_obj"],
                                                 fi["safety_d"], fi["obj_dist"], fi["obj_pos"], n_pts=n_pts)
    print("follow vx mean", float(np.mean(fx)), "too close", int(ftc.sum()), "vel bound", int(fvb.sum()))
# brake prefixes (k_brakeprefix): ragged paths and courses with per-point friction, then constant friction; about half
# of the paths brake, the memory differs from gg_scale
bv = VelocityPlanner(device="cuda:0")
bv.update_dyn_parameters(vel_max=30.0, gg_scale=0.9, ax_max_machines=g["ax_max_machines"])
brng = np.random.default_rng(8)
bplan = np.where(brng.random(70) < 0.5, brng.uniform(31.0, 70.0, size=70), brng.uniform(0.0, 30.0, size=70))
for gg, n_pts in ((fgg, np.random.default_rng(9).integers(2, 91, size=70)), ((5.0, 5.0), None)):
    bold = brng.uniform(0.5, 1.0, size=70)
    bx, bn, bi, bs = bv.check_brake_prefix(bplan, brng.uniform(10.0, 60.0, size=(70, 4)), fi["kappa"], fi["el"], gg,
                                           bold, n_course=brng.integers(0, 5, size=70), n_pts=n_pts)
    print("brake prefix mean", float(np.mean(bx)), "braking", int((bi > 0).sum()), "n_prefix", int(bn.sum()))

# positions on polylines: each mode on ragged per-query rows with invalid ones (device lengths out of range, a NaN
# position, an all-NaN row) and on a shared line
from graphbasedlocaltrajectoryplanner_b200 import pathcoord  # noqa: E402
prng = np.random.default_rng(10)
pts = torch.as_tensor(np.cumsum(prng.uniform(0.1, 2.0, size=(40, 60, 2)), axis=1), device="cuda:0")
ppos = pts[:, 20, :] + torch.as_tensor(prng.normal(0.0, 1.0, size=(40, 2)), device="cuda:0")
ppos[3, 0] = float("nan")
pts[5] = float("nan")
pn = torch.as_tensor(prng.integers(2, 61, size=40), dtype=torch.int32, device="cuda:0")
pn[0], pn[1], pn[2] = 0, 1, 61
ps, pci = pathcoord.get_s_coord(pts, ppos, n_pts=pn, closed=True)
ps2, _ = pathcoord.get_s_coord(pts, ppos, s_array=pts[:, :, 0], n_pts=pn)
pidx = pathcoord.closest_path_index(pts[0], ppos)
pin = pathcoord.check_inside_bounds(pts, pts + 2.0, ppos, n_pts=pn)
print("path coord s", float(torch.nansum(ps)), float(torch.nansum(ps2)), "idx", int(pidx.sum()), "inside",
      int(pin.sum()), "pairs", int(pci.sum()))
