"""large parity sweep (GPU box): CUDA path vs the oracle over thousands of seeded scenarios per lattice, compared with the
rules of tests/helpers.compare_records (node sequences bit-exact, coordinates / velocities 1e-4).  The oracle runs in a
process pool on the host cores.   python tests/tools/gpu_parity_sweep.py [n_per_lattice] [lattice ...] [--features]"""
import os, sys, time
REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)
import numpy as np

_W = {}


def _init(tag):
    os.environ['OPENBLAS_NUM_THREADS'] = '1'
    from tests import helpers as H
    from oracle.ltpl_oracle import OracleLTPL
    import bench
    _W['H'] = H
    _W['orc'] = OracleLTPL(bench.get_lattice(tag))
    _W['vk'] = bench.vel_kwargs()


def _work(args):
    idx, pos, heading, vel, ols, recs, zones, emerg = args
    H, orc, vk = _W['H'], _W['orc'], dict(_W['vk'], incl_emerg_traj=emerg)
    bad, ties, acts = [], 0, 0
    for i in range(len(idx)):
        want = orc.tick(pos[i], heading[i], vel[i], ols[i], vk, blocked_zones=zones[i])
        got = recs[i]
        try:
            if emerg and not want["out_of_track"]:   # 'emergency' has no full-length counterpart on the device
                em_w = want["traj"].pop("emergency", None)
                want["traj_full"].pop("emergency", None)
                id_w = want["ids"].pop("emergency", None)
                em_g = got.get("traj", {}).pop("emergency", None)
                id_g = got.get("ids", {}).pop("emergency", None)
                assert (em_w is None) == (em_g is None), "scenario %d emergency presence" % idx[i]
                if em_w is not None:
                    assert id_w % 10 == id_g % 10
                    H.assert_close("traj[emergency]", em_g[0], em_w[0], ("s", "x", "y", "psi", "kappa", "vx", "ax"),
                                   "scenario %d" % idx[i], w_rel=H.W_REL_BRAKE)
            H.compare_records(got, want, ctx="scenario %d" % idx[i])
        except AssertionError as e:
            bad.append(str(e).split("\n")[0][:300])
        if not want["out_of_track"]:
            acts += len(want["paths"])
            ties += sum(1 for a in want.get("tie", {}) if want["tie"][a] or got.get("tie", {}).get(a))
    return bad, ties, acts


def main():
    import multiprocessing as mp
    import bench
    from graphbasedlocaltrajectoryplanner_b200.planner import BatchPlanner
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    features = "--features" in sys.argv   # random blocked zones, explicit prediction arrays, emergency trajectory
    n = int(args[0]) if args else 4000
    tags = args[1:] or ["l216", "default", "l430"]
    total_bad = 0
    for tag in tags:
        sc = bench.make_batch(tag, n, seed=bench.SEED + 17)
        lat = bench.get_lattice(tag)
        zones = [None] * n
        if features:
            from oracle.gen_golden import make_zone
            rng = np.random.default_rng(99)
            zones = [({"z%d" % i: make_zone(lat, rng, sc.pos[i])} if rng.random() < 0.5 else None) for i in range(n)]
            sc.set_zones(zones)
            kp = 5
            sc.pred = np.zeros((n, sc.obj.shape[1], kp, 2))
            sc.n_pred = np.full((n, sc.obj.shape[1]), -1, dtype=np.int32)
            for i in range(n):
                for k in range(int(sc.n_obj[i])):
                    if rng.random() < 0.5:
                        continue
                    m = int(rng.integers(0, kp + 1))
                    x, y, th, v, _ = sc.obj[i, k]
                    for j in range(m):
                        t = 0.25 * (j + 1)
                        sc.pred[i, k, j] = [x - np.sin(th) * v * t, y + np.cos(th) * v * t]
                    sc.n_pred[i, k] = m
        pl = BatchPlanner(lat, device="cuda:0")
        pl.set_vel_params(incl_emerg_traj=features, **bench.vel_kwargs())
        pl.stage_scenarios(sc); pl.upload(); pl.set_startpos(); pl.tick()
        t0 = time.time()
        recs = pl.records()
        chunks = []
        step = 40
        for a in range(0, n, step):
            b = min(a + step, n)
            chunks.append((list(range(a, b)), sc.pos[a:b], sc.heading[a:b], sc.vel[a:b],
                           [sc.object_list(i) for i in range(a, b)], recs[a:b], zones[a:b], features))
        ctx = mp.get_context("spawn")
        with ctx.Pool(min(bench.usable_cores(), 96), initializer=_init, initargs=(tag,)) as pool:
            res = pool.map(_work, chunks)
        bad = [m for r in res for m in r[0]]
        ties = sum(r[1] for r in res)
        acts = sum(r[2] for r in res)
        total_bad += len(bad)
        print("[%s%s] %d scenarios, %d action paths compared, %d tie-flagged (skipped), %d mismatches  (%.1f s)" %
              (tag, " +zones/predictions/emergency" if features else "", n, acts, ties, len(bad), time.time() - t0))
        for m in bad[:8]:
            print("   ", m)
    print("TOTAL mismatches:", total_bad)


if __name__ == "__main__":
    main()
