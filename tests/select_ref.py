"""NumPy restatement of the selection rule of ltpl_select_batch (csrc/ltpl_select.cuh), the reference loop's step after
every tick (main_min_example.py:83-85): per scenario the first listed action the last velocity call returned."""
import numpy as np

NSLOT = 3
ACT_NONE, ACT_EMERGENCY = -1, 4


def select_ref(action_id, traj_row, traj_len, traj_id, em_info, incl_emerg, prefer):
    """action_id, traj_row, traj_len, traj_id [NSLOT][B]; em_info [B][3] (may be stale when incl_emerg is False);
    prefer [B or 1][L] integer action ids.  Returns sel_action [B] and sel_info [B][4] = (action, row, rows, id), with
    (-1, -1, 0, -1) where nothing in the list was returned."""
    B = action_id.shape[1]
    prefer = np.broadcast_to(np.asarray(prefer, dtype=np.int64), (B, np.shape(prefer)[1]))
    info = np.tile(np.array([ACT_NONE, -1, 0, -1], dtype=np.int32), (B, 1))
    for b in range(B):
        kept = bool((traj_row[:, b] >= 0).any())
        for a in prefer[b]:
            if a == ACT_EMERGENCY:
                if incl_emerg and kept and em_info[b, 0] >= 0:   # OTH:1027-1034
                    info[b] = (a, em_info[b, 0], em_info[b, 1], em_info[b, 2])
                    break
            elif 0 <= a < ACT_EMERGENCY:
                s = [s for s in range(NSLOT) if action_id[s, b] == a and traj_row[s, b] >= 0]
                if s:
                    info[b] = (a, traj_row[s[0], b], traj_len[s[0], b], traj_id[s[0], b])
                    break
    return info[:, 0].copy(), info
