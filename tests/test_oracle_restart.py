"""Restarts inside a closed loop: set_startpos on a live planner (OTH:161-179, 204: reinit_iterative_memory), followed by
a first tick with the forced 'straight'.  The session oracle with restarts (tests/restart_session.py) against sequences
of the unmodified reference (tests/golden/ticks_multitick_restart_{default,l216}.npz, tests/tools/gen_golden_restart.py),
the coverage of those fixtures, and the host-side checks of BatchPlanner's restart mask (no GPU needed)."""
import numpy as np
import pytest

from tests import helpers as H

FIXTURES = (("ticks_multitick_restart_default.npz", "default"), ("ticks_multitick_restart_l216.npz", "l216"))
KIND_A, KIND_B, KIND_OFF, KIND_HEAD = 1, 2, 3, 4


class _Clock(object):
    def __init__(self):
        self.t = 1000.0

    def __call__(self):
        return self.t


def _object_list(g, q, k):
    n_obj = int(g["sc_n_obj"][q])
    return [{'id': j + 1, 'type': 'physical', 'X': float(o[0]), 'Y': float(o[1]), 'theta': float(o[2]),
             'v': float(o[3]), 'length': float(o[4]), 'width': 2.5} for j, o in enumerate(g["obj"][q, k, :n_obj])]


@pytest.mark.parametrize("fixture,tag", FIXTURES)
def test_session_oracle_matches_reference_restarts(fixture, tag):
    """every planned tick of every sequence: node sequences, path lengths, trajectories, the emergency trajectory and the
    id pattern; a restart resets the memory but not the id counter or the calculation-time buffer"""
    from oracle.ltpl_oracle import OracleLTPL
    from tests.restart_session import RestartSession
    g = H.golden(fixture)
    lat = H.lattice_for(tag)
    vk = dict(vel_max=100.0, local_gg=(5.0, 5.0), ax_max_machines=g["ax_max_machines"], safety_d=30.0,
              incl_emerg_traj=True)
    n_seq, n_ticks = g["dt"].shape
    compared, restarted = 0, 0
    for q in range(n_seq):
        clock = _Clock()
        ses = RestartSession(OracleLTPL(lat), clock=clock)
        for k in range(n_ticks):
            ctx = "sequence %d tick %d" % (q, k)
            clock.t += float(g["dt"][q, k])
            if k == 0 or g["restart"][q, k]:
                rejected = ses.set_startpos(g["pos"][q, k], g["heading"][q, k], g["vel"][q, k])
                assert rejected == bool(g["rejected"][q, k]), ctx + " rejected"
                restarted += int(k > 0 and not rejected)
            if not g["planned"][q, k]:
                continue
            sel = (H.ACTIONS + ("emergency",))[int(g["sel"][q, k])]
            paths = ses.calc_paths(sel, _object_list(g, q, k))
            for a, act in enumerate(H.ACTIONS):
                n_want = int(g["path_len"][q, k, a])
                assert (act in paths) == (n_want > 0), "%s: path %s" % (ctx, act)
                if n_want:
                    assert paths[act][0].shape[0] == n_want, ctx + " path length " + act
                    nd = [[-1 if v is None else int(v) for v in p] for p in ses.m_nodes[act][0]]
                    assert nd == g["nodes"][q, k, a, :int(g["nodes_len"][q, k, a])].tolist(), ctx + " nodes " + act
            base = ses.traj_base_id
            traj, ids = ses.calc_vel_profile(g["pos"][q, k], float(g["vel_est"][q, k]),
                                             **dict(vk, gg_scale=float(g["gg_scale"][q, k])))
            assert ses.traj_base_id == base + 10
            for a, act in enumerate(H.ACTIONS):
                t_want = int(g["traj_len"][q, k, a])
                assert (act in traj) == (t_want > 0), "%s: trajectory %s" % (ctx, act)
                if t_want:
                    assert ids[act] % 10 == int(g["traj_id"][q, k, a]) % 10, ctx + " id " + act
                    H.assert_close("traj[%s]" % act, traj[act][0], g["traj"][q, k, a, :t_want],
                                   ("s", "x", "y", "psi", "kappa", "vx", "ax"), ctx)
                    compared += 1
            n_em = int(g["em_len"][q, k])
            assert ("emergency" in traj) == (n_em > 0), ctx + " emergency"
            if n_em:
                H.assert_close("traj[emergency]", traj["emergency"][0], g["em_traj"][q, k, :n_em],
                               ("s", "x", "y", "psi", "kappa", "vx", "ax"), ctx)
    assert restarted >= 20 and compared > 120, (restarted, compared)


def test_restart_ids_keep_counting_in_the_reference():
    """the reference's id base (+10 per calc_vel_profile, OTH:669) is not reset by set_startpos: within a sequence the
    ids grow by 10 per planned tick across every restart"""
    g = H.golden(FIXTURES[0][0])
    for q in range(g["dt"].shape[0]):
        ks = [k for k in range(g["dt"].shape[1]) if g["planned"][q, k] and (g["traj_id"][q, k] >= 0).any()]
        base = [int(g["traj_id"][q, k][g["traj_id"][q, k] >= 0][0]) // 10 for k in ks]
        planned_before = [int(g["planned"][q, :k].sum()) for k in ks]
        assert [b - p for b, p in zip(base, planned_before)] == [base[0] - planned_before[0]] * len(ks), q


@pytest.mark.parametrize("fixture,tag", FIXTURES)
def test_restart_fixture_coverage(fixture, tag):
    """restarts of every kind: (a) re-anchoring at the estimate, (b) a jump with another start velocity, (c) a rejected
    pose (off the track / wrong heading) with a valid restart one or two ticks later, (d) right after ticks that executed
    'follow', 'left' / 'right', 'emergency', and right after a grip drop (brake on the backup plan)"""
    g = H.golden(fixture)
    n_seq, n_ticks = g["dt"].shape
    assert n_seq >= 12 and n_ticks >= 10
    r = g["restart"] > 0
    assert r.sum() >= 20
    kind = g["rs_kind"]
    assert ((kind == KIND_A) & r).sum() >= 4
    jumps = (kind == KIND_B) & r & (g["rejected"] == 0)
    assert jumps.sum() >= 4
    assert ((kind == KIND_OFF) & (g["rejected"] > 0)).sum() >= 1
    assert ((kind == KIND_HEAD) & (g["rejected"] > 0)).sum() >= 1
    revived = 0
    for q, k in zip(*np.nonzero(r & (g["rejected"] > 0) & (kind >= KIND_OFF))):
        assert not g["planned"][q, k]
        nxt = [d for d in (1, 2) if k + d < n_ticks and r[q, k + d] and not g["rejected"][q, k + d]]
        revived += int(bool(nxt) and g["planned"][q, k + nxt[0]])
    assert revived >= 2
    before = np.zeros_like(r)
    before[:, 1:] = g["planned"][:, :-1] > 0
    planned_restart = r & before & (g["planned"] > 0)
    for code in (1, 4):                                    # follow, emergency
        assert (planned_restart & (g["sel"] == code)).sum() >= 1, code
    assert (planned_restart & ((g["sel"] == 2) | (g["sel"] == 3))).sum() >= 1   # left / right
    drop = np.zeros_like(r)
    drop[:, 1:] = g["gg_scale"][:, :-1] < 1.0
    assert (planned_restart & drop).sum() >= 1
    # a jump changes the start velocity: the restarted tick's profiles start at the new vel
    assert (np.abs(np.diff(g["vel"], axis=1))[(r & (g["planned"] > 0))[:, 1:]] > 1.0).sum() >= 4
    # the t_const of the reference is 0 exactly where it took no constant segment: first ticks after a (re)start
    first = r | (np.arange(n_ticks)[None, :] == 0)
    assert (g["t_const"][first & (g["planned"] > 0)] == 0.0).all()
    assert (g["t_const"][~first & (g["planned"] > 0) & before] > 0.0).all()


class _Host(object):
    """BatchPlanner's host side without a device: only what the restart-mask check reads"""

    def __init__(self, batch):
        from graphbasedlocaltrajectoryplanner_b200 import capi
        self.dims = capi.Dims()
        self.dims.batch = batch


def test_restart_mask_is_checked_on_the_host():
    from graphbasedlocaltrajectoryplanner_b200.planner import BatchPlanner
    h = _Host(5)
    check = BatchPlanner._restart_mask
    assert check(h, None) is None
    assert check(h, np.zeros(5, dtype=bool)) is None                      # no entry set: NULL, today's launches
    m = check(h, [0, 1, 0, 0, 2])
    assert m.dtype == bool and m.tolist() == [False, True, False, False, True]
    for bad in (np.ones(4, dtype=bool), np.ones((5, 1), dtype=bool), np.ones((1, 5), dtype=bool), True):
        with pytest.raises(ValueError):
            check(h, bad)
