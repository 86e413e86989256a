// ltpl_state.cuh -- stateful tick (DESIGN.md section 11): the iterative memory of OnlineTrajectoryHandler
// on the device.  The memory of the reference (OTH:64-87: __last_action_set_{path_param, node_idx, nodes, coeff},
// __last_bp_action_set) IS the output of the previous tick: a second LtplBuffers set (prev_*) used ping-pong, plus three
// integers per path instead of the slicing of OTH:705-731:
//     m = first memory point   (cut_index_layer, OTH:712)      path-plane index
//     L = first memory node    (cut_layer,       OTH:586)      node index
//     c = first trajectory row (cut_index_pos,   OTH:578)      path-plane index;  __last_cut_idx = c - m (OTH:598)
// The exported trajectory ("bp", <= n_export rows because LTPL:401-406 cuts the dict it shares with the handler) is
// rows 0 .. traj_len-1 of the previous s / vx planes, its x, y are path-plane points c .. c + traj_len - 1.
//
// k_state  (warp / scenario, replaces k_startpos from the second tick on): OTH:346-392 -- index on the last executed
//          trajectory reached after t_const, next node behind it = start node of the search, constant segment = memory
//          path up to that node, the <= 3 first edges of the remaining last solution get the cost factors of GLNT:155-162.
// k_ref    (warp / scenario, between k_path and the velocity kernel): OTH:518-601 get_ref_idx -- cut index from the
//          position estimate, delay compensation (vel_plan, vel_course), cut layer from the NEW node index list; also the
//          follow-mode object distance on the cut follow path (OTH:774-784).
// k_prefix (warp / path, after the velocity kernel): vel_course in front of the profile (OTH:826, 915), arc length from the
//          cut, ax across the seam, exported row count.
#pragma once
#include "ltpl_plan.cuh"


// get_s_coord(..., only_index=True)[1] on an OPEN polyline given by a gather pt(i), i < n (get_s_coord.py:40-58, 94-97):
// nearest point (first minimum), then the neighbour on the side of the larger angle; returns the pair (i0, i1)
template <class PT>
__device__ __forceinline__ int2 open_index_pair(PT pt, int n, double px, double py, int lane) {
    double bv = LTPL_INF;
    int bi = 0x7fffffff;
    for (int j = lane; j < n; j += 32) {
        const double2 p = pt(j);
        const double d = dist2_rn(p.x, p.y, px, py);
        if (d < bv) {
            bv = d;
            bi = j;
        }
    }
    const int nb = warp_argmin(bv, bi).i;
    const int idx1 = max(nb - 1, 0), idx2 = min(nb + 1, n - 1);
    return angle_cmp(pt(nb), px, py, pt(idx1), pt(idx2)).ge ? make_int2(idx1, nb) : make_int2(nb, idx2);
}

// lattice edge (start layer, src node) -> (next layer, dst node), or -1 (GB.get_eid on the filtered graph, GB:505-511)
__device__ __forceinline__ int find_edge(const LatDev& lt, int layer, int src, int nxt_layer, int dst) {
    if (layer < 0 || nxt_layer < 0) return -1;
    const int2 io = lt.in_off[lt.node_off[nxt_layer] + dst];
    for (int k = 0; k < io.y; ++k)
        if (lt.edge_src[io.x + k] == src) {
            // in-edges of a node all start in the previous layer; make sure it is the right one (closed tracks wrap)
            const int e = io.x + k;
            return (e >= lt.edge_layer_off[layer] && e < lt.edge_layer_off[layer + 1]) ? e : -1;
        }
    return -1;
}

__global__ void __launch_bounds__(LTPL_WARPS_PER_CTA * 32)
k_state(const __grid_constant__ LatDev lt, const __grid_constant__ LtplParams prm,
        const __grid_constant__ LtplDims dm, const __grid_constant__ LtplBuffers bf) {
    const int lane = threadIdx.x & 31;
    const int b = sub_scenario(dm, LTPL_WARPS_PER_CTA);
    if (b < 0) return;
    const int B = dm.batch;
    int* info = bf.st_info + 8 * (size_t)b;
    if (bf.restart && bf.restart[b]) {
        // set_startpos on the live instance (OTH:161-179, 204): k_startpos has just checked the pose and seeded the forced
        // 'straight' segment; the memory is dropped.  Marker for the later kernels: st_info[0] = -1 -- the constant
        // segment is set_startpos's, no cost reduction, cut 0 at vel (get_ref_idx without a last trajectory, OTH:592-598),
        // no backup plan.  A rejected pose keeps the flags k_startpos wrote.
        if (lane == 0 && bf.sc_flags[b] == 0) {
            info[0] = -1;
            info[1] = info[2] = 0;
            info[3] = 1;                                 // the leading (-1, -1) entry
            info[4] = 0;
            info[5] = info[6] = info[7] = -1;
            bf.vel_plan[b] = bf.vel[b];
        }
        return;
    }
    // a scenario whose start pose was rejected (set_startpos returned True, LTPL:268-298) stays so until it is re-anchored
    const int old_flags = bf.sc_flags[b];
    if (old_flags & (LTPL_SC_OUT_OF_TRACK | LTPL_SC_HEADING_MISMATCH)) return;
    const int old_sl = bf.start_node[2 * b], old_sn = bf.start_node[2 * b + 1];   // start node of the last tick (OTH:393-407)
    __syncwarp();
    if (lane == 0) {
        bf.start_node[2 * b] = -1;
        bf.start_node[2 * b + 1] = -1;
        bf.const_len[b] = 0;
    }
    // the executed action (OTH:307-315); 'emergency' stands for the action its profile was based on = the first kept
    // trajectory of the last tick (OTH:1027-1030, k_emergency), provided that tick had an emergency trajectory
    int sel = bf.sel_action[b];
    if (sel == LTPL_ACT_EMERGENCY) {
        sel = LTPL_ACT_NONE;
        if (bf.prev_em_info && bf.prev_em_vx && bf.prev_em_info[3 * (size_t)b] >= 0)
            for (int s = LTPL_NSLOT - 1; s >= 0; --s)
                if (bf.prev_traj_len[s * B + b] > 0) sel = bf.prev_action_id[s * B + b];
    }
    int qp = -1;
    for (int s = 0; s < LTPL_NSLOT; ++s)
        if (bf.prev_action_id[s * B + b] == sel && sel != LTPL_ACT_NONE) qp = s * B + b;
    // an action set removed by the velocity planner (OTH:1007-1025) was popped from the memory dicts as well
    if (qp >= 0 && bf.prev_traj_len[qp] == 0) qp = -1;
    const int nb_rows = (qp >= 0) ? bf.prev_traj_len[qp] : 0;
    if (qp < 0 && old_flags == 0 && old_sl >= 0) {
        // OTH:393-407 with an executed action the last tick did not return (no constant segment, OTH:409-411): the search
        // starts at the OLD start node again, nothing is stitched (OTH:433-472 skipped), no cost reduction (GLNT:155), no
        // backup plan (OTH:339-344), and get_ref_idx falls back to the initial velocity (OTH:592-598: cut 0, v_start).
        // Marker for the later kernels: const_len == 0.
        if (lane == 0) {
            bf.sc_flags[b] = 0;
            bf.start_node[2 * b] = old_sl;
            bf.start_node[2 * b + 1] = old_sn;
            bf.const_len[b] = 0;
            info[0] = b;                                 // a valid row; nothing of it is used (cnd = 0, const_len = 0)
            info[1] = 0;
            info[2] = 0;
            info[3] = 0;
            info[4] = 0;
            info[5] = info[6] = info[7] = -1;
            bf.vel_plan[b] = bf.vel[b];                  // `vel` of a stateful tick = v_start of set_startpos (OTH:597)
        }
        return;
    }
    if (qp < 0 || nb_rows <= 2) {   // OTH:319-322, constant segment exists but <= 2 trajectory rows: not planned
        if (lane == 0) bf.sc_flags[b] = LTPL_SC_STATE_FALLBACK | ((qp < 0 ? 1 : 2) << LTPL_SC_REASON_SHIFT);
        return;
    }
    const int m_p = bf.prev_trim[4 * qp + 0], L_p = bf.prev_trim[4 * qp + 1], c_p = bf.prev_trim[4 * qp + 2];
    const size_t pplane = (size_t)LTPL_NSLOT * B * dm.p_max;
    const double* Px = bf.prev_path + (size_t)qp * dm.p_max;
    const double* Py = Px + pplane;
    const double* S = bf.prev_s_vx_ax + (size_t)qp * dm.p_max;
    const double* V = S + pplane;

    // index of the pose on the last trajectory after t_const (OTH:366-378; quirk q11: ds / v with inf where v == 0)
    int next_idx = 1;
    if (lane == 0) {
        const double t_const = bf.t_const[b];
        double cum = 0.0;
        int arg = 0;
        for (int i = 0; i + 2 < nb_rows; ++i) {   // j = i + 1: (s[j + 1] - s[j]) / v[j]
            const double v = V[i + 1];
            const double t = (v != 0.0) ? __ddiv_rn(__dsub_rn(S[i + 2], S[i + 1]), v) : LTPL_INF;
            cum = __dadd_rn(cum, t);
            if (!(cum <= t_const)) {
                arg = i;
                break;
            }
        }
        next_idx = arg + 1;
    }
    next_idx = __shfl_sync(LTPL_FULL, next_idx, 0);
    const double ppx = Px[c_p + next_idx], ppy = Py[c_p + next_idx];   // predicted position (OTH:383)

    // first node after the predicted position (OTH:381-386)
    const int nn_mem = bf.prev_n_nodes[qp] - L_p;   // nodes of the (trimmed) memory
    if (nn_mem < 2) {
        if (lane == 0) bf.sc_flags[b] = LTPL_SC_STATE_FALLBACK | (3 << LTPL_SC_REASON_SHIFT);
        return;
    }
    const int* Ip = bf.prev_node_idx + (size_t)qp * dm.h_max + L_p;
    const int* Np = bf.prev_nodes + ((size_t)qp * dm.h_max + L_p) * 2;
    const int2 pair = open_index_pair([&](int i) { const int pi = Ip[i]; return make_double2(Px[pi], Py[pi]); },
                                      nn_mem, ppx, ppy, lane);
    const int sni = pair.y;                          // start_node_idx within the memory node list
    const int loc = Ip[sni] - m_p;                   // loc_path_start_idx within the memory path
    const int sl = Np[2 * sni], sn = Np[2 * sni + 1];
    if (sl < 0 || loc + 1 > dm.p_max) {
        if (lane == 0) bf.sc_flags[b] = LTPL_SC_STATE_FALLBACK | ((sl < 0 ? 4 : 5) << LTPL_SC_REASON_SHIFT);
        return;
    }
    if (lane == 0) {
        bf.sc_flags[b] = 0;
        bf.start_node[2 * b] = sl;
        bf.start_node[2 * b + 1] = sn;
        bf.const_len[b] = loc + 1;
        info[0] = qp;
        info[1] = m_p;
        info[2] = L_p;
        info[3] = sni;                               // number of constant nodes in front of the start node
        // cost reduction on the first edges of the remaining last solution (GLNT:155-162)
        int n_fe = 0;
        for (int i = 0; i < 3; ++i) {
            info[5 + i] = -1;
            if (sni + i + 1 < nn_mem) {
                const int e = find_edge(lt, Np[2 * (sni + i)], Np[2 * (sni + i) + 1], Np[2 * (sni + i + 1)],
                                        Np[2 * (sni + i + 1) + 1]);
                info[5 + i] = e;   // slot i keeps factor w_last_edges[i]; -1: edge not in the lattice
                n_fe = i + 1;
            }
        }
        info[4] = n_fe;
    }
}

// follow mode: distance to the closest object along the cut follow path (OTH:766-784); no object -> 0 (OTH:766-768)
__device__ __forceinline__ void ref_obj_dist(const LtplDims& dm, const LtplBuffers& bf, int b, int cut_pos, double px,
                                             double py, int lane) {
    const int B = dm.batch;
    const size_t pplane = (size_t)LTPL_NSLOT * B * dm.p_max;
    if (lane == 0) bf.obj_dist[b] = 0.0;
    __syncwarp();
    const int qf = b;   // slot 0
    if (bf.action_id[qf] == LTPL_ACT_FOLLOW && bf.closest_obj[b] >= 0) {
        const int n = bf.path_len[qf] - cut_pos;
        const double* X = bf.path + (size_t)qf * dm.p_max + cut_pos;
        const double* Y = X + pplane;
        const double* E = X + 4 * pplane;
        double s_two[2];
#pragma unroll 1
        for (int w = 0; w < 2; ++w) {
            const double tx = w ? px : bf.cobj[4 * b], ty = w ? py : bf.cobj[4 * b + 1];
            double v2 = LTPL_INF;
            int i2 = 0x7fffffff;
            for (int j = lane; j < n; j += 32) {
                const double d = dist2_rn(X[j], Y[j], tx, ty);
                if (d < v2) {
                    v2 = d;
                    i2 = j;
                }
            }
            const int nbp = warp_argmin(v2, i2).i;
            const int i1 = max(nbp - 1, 0), j2 = min(nbp + 1, n - 1);
            const bool gt = angle_cmp(make_double2(X[nbp], Y[nbp]), tx, ty, make_double2(X[i1], Y[i1]),
                                      make_double2(X[j2], Y[j2])).gt;
            const int ia = gt ? i1 : nbp, ib = gt ? nbp : j2;
            // s_array = cumsum(el) of the cut path; leading 0 inserted when el[0] > 0.05 (get_s_coord.py:67-68)
            double acc = 0.0;                        // cumsum(el)[ia - 1 + ins] evaluated by lane 0 order of np.cumsum
            const bool ins = E[0] > 0.05;
            const int upto = ins ? ia : ia + 1;      // number of el terms summed
            for (int j = 0; j < upto; ++j) acc = __dadd_rn(acc, E[j]);
            const double ax_ = X[ia], ay_ = Y[ia], bx = X[ib] - ax_, by = Y[ib] - ay_;
            const double t = __ddiv_rn(__dadd_rn(__dmul_rn(tx - ax_, bx), __dmul_rn(ty - ay_, by)),
                                       __dadd_rn(sq_rn(bx), sq_rn(by)));
            const double sx = __dadd_rn(ax_, __dmul_rn(t, bx)), sy = __dadd_rn(ay_, __dmul_rn(t, by));
            s_two[w] = __dadd_rn(acc, sqrt(__dadd_rn(sq_rn(ax_ - sx), sq_rn(ay_ - sy))));
        }
        if (lane == 0) bf.obj_dist[b] = s_two[0] - s_two[1];
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// k_ref: get_ref_idx (OTH:518-601) + follow-mode object distance (OTH:774-784)
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(LTPL_WARPS_PER_CTA * 32)
k_ref(const __grid_constant__ LatDev lt, const __grid_constant__ LtplParams prm,
      const __grid_constant__ LtplDims dm, const __grid_constant__ LtplBuffers bf) {
    const int lane = threadIdx.x & 31;
    const int b = sub_scenario(dm, LTPL_WARPS_PER_CTA);
    if (b < 0) return;
    const int B = dm.batch;
    if (bf.sc_flags[b] != 0) return;
    const int* info = bf.st_info + 8 * (size_t)b;
    if (bf.const_len[b] == 0 || info[0] < 0) {   // OTH:592-598: no valid last solution (or a restart) -> cut 0, no
                                                 // vel_course, vel_plan = v_start (k_state)
        if (lane < LTPL_NSLOT) {
            int* tr = bf.trim + 4 * (size_t)(lane * B + b);
            tr[0] = tr[1] = tr[2] = tr[3] = 0;
        }
        __syncwarp();
        ref_obj_dist(dm, bf, b, 0, bf.pos[2 * b], bf.pos[2 * b + 1], lane);
        return;
    }
    const int qp = info[0], m_p = info[1];
    const int c_p = bf.prev_trim[4 * qp + 2];
    const int nb_rows = bf.prev_traj_len[qp];
    const size_t pplane = (size_t)LTPL_NSLOT * B * dm.p_max;
    const double* Px = bf.prev_path + (size_t)qp * dm.p_max + c_p;   // trajectory row j -> path point c + j
    const double* Py = Px + pplane;
    const double* S = bf.prev_s_vx_ax + (size_t)qp * dm.p_max;
    const double* V = S + pplane;
    // an executed 'emergency' trajectory shares s, x, y with its base (calc_brake_emergency.py:40-45) but not the velocity
    if (bf.sel_action[b] == LTPL_ACT_EMERGENCY) V = bf.prev_em_vx + (size_t)b * dm.n_export;
    const double px = bf.pos[2 * b], py = bf.pos[2 * b + 1];

    // cut index: first of the two trajectory points around pos_est (OTH:551-556); n_export <= 128 rows
    double bv = LTPL_INF;
    int bi = 0x7fffffff;
    for (int j = lane; j < nb_rows; j += 32) {
        const double d = dist2_rn(Px[j], Py[j], px, py);
        if (d < bv) {
            bv = d;
            bi = j;
        }
    }
    const ArgMinD mm = warp_argmin(bv, bi);
    const int nb = mm.i;
    const int idx1 = max(nb - 1, 0), idx2 = min(nb + 1, nb_rows - 1);
    const AngCmp ac = angle_cmp(make_double2(Px[nb], Py[nb]), px, py, make_double2(Px[idx1], Py[idx1]),
                                make_double2(Px[idx2], Py[idx2]));
    const int cut_index = ac.ge ? idx1 : nb;

    // delay compensation (OTH:558-574)
    int vel_idx = 1;
    if (lane == 0) {
        double cum = 0.0;
        int arg = 0;
        const int nv = nb_rows - 1 - cut_index;      // v_past = bp[cut:-1, 5]
        for (int i = 0; i < nv; ++i) {
            const double v = V[cut_index + i];
            const double t = (v != 0.0) ? __ddiv_rn(__dsub_rn(S[cut_index + i + 1], S[cut_index + i]), v) : LTPL_INF;
            cum = __dadd_rn(cum, t);
            if (!(cum <= prm.delaycomp)) {
                arg = i;
                break;
            }
        }
        vel_idx = min(arg + 1, nv - 1);   // -1: the cut is the LAST row of the last trajectory -- v_past is empty
        if (vel_idx >= 0) {
            bf.vel_plan[b] = V[cut_index + vel_idx];
            // `course` holds n_export rows per scenario = as many as an exported trajectory has: no truncation
            for (int i = 0; i < vel_idx; ++i) bf.course[(size_t)b * dm.n_export + i] = V[cut_index + i];
        }
    }
    vel_idx = __shfl_sync(LTPL_FULL, vel_idx, 0);
    if (vel_idx < 0) {   // np.argmin of an empty array raises in the reference (OTH:570): not planned, re-anchor
        if (lane == 0) bf.sc_flags[b] = LTPL_SC_STATE_FALLBACK | (7 << LTPL_SC_REASON_SHIFT);
        return;
    }
    const int cut_pos = (c_p - m_p) + cut_index;     // cut_index_pos in the NEW path planes (OTH:577)

    // cut layer from the node index list of the first action of this tick (OTH:580-590)
    int q0 = -1;
    for (int s = LTPL_NSLOT - 1; s >= 0; --s)
        if (bf.action_id[s * B + b] != LTPL_ACT_NONE) q0 = s * B + b;
    int cut_layer = 0;
    if (q0 >= 0) {
        const int nn = bf.n_nodes[q0];
        const int* ni = bf.node_idx + (size_t)q0 * dm.h_max;
        int first = nn;                              // np.argmin(node_idx < cut_pos): first index with node_idx >= cut_pos
        for (int i = lane; i < nn; i += 32)
            if (!(ni[i] < cut_pos)) first = min(first, i);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) first = min(first, __shfl_xor_sync(LTPL_FULL, first, o));
        if (first == nn) first = 0;                  // all True -> argmin = 0
        cut_layer = max(first - 2, 0);
    }
    if (lane < LTPL_NSLOT) {
        const int q = lane * B + b;
        int* tr = bf.trim + 4 * (size_t)q;
        if (bf.action_id[q] != LTPL_ACT_NONE) {
            tr[0] = bf.node_idx[(size_t)q * dm.h_max + cut_layer];
            tr[1] = cut_layer;
            tr[2] = cut_pos;
            tr[3] = vel_idx;
        } else {
            tr[0] = tr[1] = tr[2] = tr[3] = 0;
        }
    }

    ref_obj_dist(dm, bf, b, cut_pos, px, py, lane);
}

// ---------------------------------------------------------------------------------------------------------------------
// k_prefix: the velocity kernel of a stateful tick works on the path behind the cut AND behind vel_course (rows pref ..
// of the s / vx / ax planes, arc length 0 at its first point).  This kernel puts vel_course in front (OTH:826, 915),
// shifts the arc length to 0 at the cut (OTH:743), computes ax across the seam (OTH:935-939) and sets the row count.
// One warp per path.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(LTPL_WARPS_PER_CTA * 32)
k_prefix(const __grid_constant__ LtplDims dm, const __grid_constant__ LtplBuffers bf) {
    const int lane = threadIdx.x & 31;
    const int B = dm.batch;
    const int q = sub_path(dm, LTPL_WARPS_PER_CTA);
    if (q < 0) return;
    if (!(bf.status[q] & LTPL_ST_TRAJ_VALID)) return;
    const int b = q % B;
    const int cut = bf.trim[4 * q + 2], pref = bf.trim[4 * q + 3];
    const int n_p = bf.path_len[q] - cut - pref;             // points the velocity kernel worked on
    const size_t pplane = (size_t)LTPL_NSLOT * B * dm.p_max;
    const double* E = bf.path + 4 * pplane + (size_t)q * dm.p_max + cut;
    double* S = bf.s_vx_ax + (size_t)q * dm.p_max;
    double* VX = S + pplane;
    double* AX = VX + pplane;
    double s_pref = 0.0;
    for (int j = 0; j < pref; ++j) s_pref = __dadd_rn(s_pref, E[j]);
    for (int i = pref + lane; i < pref + n_p; i += 32) S[i] += s_pref;
    __syncwarp();
    if (lane == 0) {
        double acc = 0.0;
        for (int i = 0; i < pref; ++i) {
            S[i] = acc;
            VX[i] = bf.course[(size_t)b * dm.n_export + i];
            acc = __dadd_rn(acc, E[i]);
        }
        for (int i = 0; i < pref; ++i) {
            const double v0 = VX[i], v1 = VX[i + 1];
            double a = (v1 * v1 - v0 * v0) / (2 * (S[i + 1] - S[i]));
            if (fabs(v0) <= 1e-8 && fabs(a) <= 1e-8) a = -5.0;   // np.isclose(vx, 0) & np.isclose(ax, 0) (OTH:939)
            AX[i] = a;
        }
        bf.traj_len[q] = min(n_p + pref, dm.n_export);
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// k_backup: recursive infeasibility (OTH:950-1006).  A straight / follow profile of a stateful tick that cannot start at
// the planned velocity (e.g. the grip dropped) is replaced by full braking on the BACKUP plan = the memory of the last
// tick's follow / straight path (OTH:325-344; both live in slot 0): the path, node and coefficient lists of this tick
// become the backup's (OTH:958-963), the trajectory is vel_course followed by tph.calc_vel_profile_brake on the backup
// path behind it with the caller's local_gg WITHOUT gg_scale (VPFB:229-255, OTH:965-1003).  One warp per scenario, between
// the velocity kernel and k_prefix (which adds vel_course, the arc-length offset and the row count as for every path).
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(LTPL_WARPS_PER_CTA * 32)
k_backup(const __grid_constant__ LtplParams prm, const __grid_constant__ LtplDims dm, const __grid_constant__ LtplBuffers bf) {
    const int lane = threadIdx.x & 31;
    const int b = sub_scenario(dm, LTPL_WARPS_PER_CTA);
    if (b < 0) return;
    const int B = dm.batch;
    const int q = b;   // slot 0: follow / straight
    const int st = bf.status[q];
    const int act = bf.action_id[q];
    if (!(st & LTPL_ST_TRAJ_VALID) || !(st & LTPL_ST_VEL_BOUND_VIOL) ||
        !(act == LTPL_ACT_FOLLOW || act == LTPL_ACT_STRAIGHT))
        return;
    if (bf.const_len[b] == 0 || bf.st_info[8 * (size_t)b] < 0) return;   // invalid last solution or restart: no backup
                                                                         // plan (OTH:339-344)
    const int pa = bf.prev_action_id[q];
    if (!(pa == LTPL_ACT_FOLLOW || pa == LTPL_ACT_STRAIGHT)) return;   // no backup plan: stays flagged
    const int m_b = bf.prev_trim[4 * q + 0], L_b = bf.prev_trim[4 * q + 1];
    const int n_bk = bf.prev_path_len[q] - m_b, nn_bk = bf.prev_n_nodes[q] - L_b;
    const int cut = bf.trim[4 * q + 2], pref = bf.trim[4 * q + 3];
    const int n_p = n_bk - cut - pref;                     // points of the brake profile
    if (n_p < 1 || nn_bk < 1) return;
    const size_t pplane = (size_t)LTPL_NSLOT * B * dm.p_max;
    // the backup becomes this tick's memory (OTH:958-963); the trims of k_ref stay (they are what the slices use)
    for (int c = 0; c < 5; ++c) {
        const double* src = bf.prev_path + c * pplane + (size_t)q * dm.p_max + m_b;
        double* dst = bf.path + c * pplane + (size_t)q * dm.p_max;
        for (int i = lane; i < n_bk; i += 32) dst[i] = src[i];
    }
    for (int j = lane; j < nn_bk; j += 32) {
        bf.node_idx[(size_t)q * dm.h_max + j] = bf.prev_node_idx[(size_t)q * dm.h_max + L_b + j] - m_b;
        bf.nodes[((size_t)q * dm.h_max + j) * 2] = bf.prev_nodes[((size_t)q * dm.h_max + L_b + j) * 2];
        bf.nodes[((size_t)q * dm.h_max + j) * 2 + 1] = bf.prev_nodes[((size_t)q * dm.h_max + L_b + j) * 2 + 1];
    }
    for (int j = lane; j < max(nn_bk - 1, 1) * 8; j += 32)
        bf.coeff[(size_t)q * dm.h_max * 8 + j] = bf.prev_coeff[((size_t)q * dm.h_max + L_b) * 8 + j];
    __syncwarp();
    if (lane == 0) {
        bf.path_len[q] = n_bk;
        bf.n_nodes[q] = nn_bk;
        // full braking from the planned velocity behind vel_course (tph.calc_vel_profile_brake, mode 'decel_forw')
        const double* K = bf.path + 3 * pplane + (size_t)q * dm.p_max + cut + pref;
        const double* E = K + pplane;
        double* S = bf.s_vx_ax + (size_t)q * dm.p_max + pref;   // rows behind vel_course, arc length 0 at their first point
        double* VX = S + pplane;
        double* AX = VX + pplane;
        const double dmq = prm.drag_coeff / prm.m_veh, inv_ay = 1.0 / prm.gg_ay;
        // location dependent local_gg of the LAST tick along the backup path (__backup_path_gg, OTH:970-975), raw
        const double* ggr = bf.prev_gg ? bf.prev_gg + (size_t)q * dm.p_max + m_b + cut + pref : nullptr;
        double v0 = bf.vel[b];                                  // == vel_plan (run_tick launches k_backup so)
        if (v0 < 0.0) v0 = 0.0;
        double w = v0 * v0, s = 0.0;
        bool stopped = false;
        for (int i = 0; i < n_p; ++i) {
            S[i] = s;
            VX[i] = sqrt(w);
            double wn = 0.0;
            if (i + 1 < n_p) {
                if (!stopped) {
                    const double a = ggr ? acc_brake(w, fabs(K[i]), ggr[i], 1.0 / ggr[pplane + i], prm.dyn_model_exp, dmq)
                                         : acc_brake(w, fabs(K[i]), prm.gg_ax, inv_ay, prm.dyn_model_exp, dmq);
                    const double nx = fma(2.0 * a, E[i], w);
                    if (nx < 0.0)
                        stopped = true;
                    else
                        wn = nx;
                }
                double ax = (wn - w) / (2 * E[i]);
                if (w <= 1e-16 && fabs(ax) <= 1e-8) ax = -5.0;   // OTH:999
                AX[i] = ax;
                s = __dadd_rn(s, E[i]);
            } else {
                AX[i] = 0.0;
            }
            w = wn;
        }
        bf.traj_len[q] = min(n_p, dm.n_export);                 // k_prefix adds the vel_course rows
        atomicAnd(&bf.sc_flags[b], ~(LTPL_SC_STATE_FALLBACK | (7 << LTPL_SC_REASON_SHIFT)));    // handled
    }
}
