// ltpl_velfollow.cuh -- stand-alone follow-mode velocity profiles over the caller's paths (ltpl_vel_follow_batch):
//   k_velfollow   VpForwardBackward.calc_vel_profile_follow (VPFB:141-192) -> calc_vel_profile_follow (CVPF:78-313)
//
// The arithmetic is the tick's follow path (k_vel_res, DESIGN.md sections 5 and 6) on the tiling of k_velprofile: one LANE
// per path, one warp = 32 paths, the path arrays stream through shared memory in tiles of VD_H points x 32 paths
// (ltpl_velprofile.cuh).  Per path, in CVPF's order:
//   0. the opponent (once per lane, no path array): nearest race-line point to obj_pos (first minimum of the squared
//      distances), the closed get_s_coord neighbour rule (index -1 wraps), then its float64 brake chain over the rolled
//      race line with ggv = [100, 14, 14] until v <= 0.1 m/s (opp_stop_dist).  The race line's x, y sit in shared memory
//      when they fit into the tile area (which is idle during this phase), else every lane reads them through L2 (all lanes
//      of the warp read the same point: one broadcast load)
//   1. pass F1 (forward): s = cumsum(el), stop_idx, the float64 ego brake profile (brake_step, the step of k_velbrake) with
//      its indices id_brake (v <= 0.1) and argmax(v <= v_control); v_ego_brake goes to the caller's vx row.  The pass ends
//      as soon as every lane of the warp has stopped braking and passed s_stop
//   2. pass F2 (forward): the complete profile on [0, n - 1] and the control profile on [idx_c, stop_idx] (VRSweep::fwd,
//      fp32 in w = v^2), both w rows as one float pair per point in the caller's ax row
//   3. pass B (backward): both backward sweeps (VRSweep::bwd), the merge min(profile, complete), vx, ax and the flags
// Every decision (nearest index, neighbour rule, stop_idx, id_brake, idx_c, ego_stop_dist < s_stop, the flags) is taken in
// float64; the two stop distances are summed in index order (as the tick does; np.sum's pairwise order differs in the
// last bits only).
// HBM traffic per point (constant friction): F1 16 B in (kappa, el) + 8 B out (brake; only up to standstill / s_stop),
// F2 16 B in + 8 B out (w pair), B 16 B in + 8 B (w pair) + 8 B (brake) in + 16 B out (vx, ax) = 96 B at most;
// per-point friction adds 16 B in F1 and F2 and 32 B in B (own and two mirrored friction pairs).
#pragma once
#include "ltpl_velprofile.cuh"

#define VF_NONE 0x7fffffff

// tile area: kappa, el, w pair, brake (+ GG: two friction tiles per profile) of VD_TILE float64 elements each
__host__ __device__ constexpr int vf_tiles(bool gg) { return gg ? 8 : 4; }
// + s_n, s_o, s_z, s_lo, s_hi, s_st, s_fb (per-row point counts, the control range, stop_idx, flag bits) and the per-lane
// float64 scalars s_dv[5][32]
__host__ __device__ constexpr int vf_smem(bool gg) { return vf_tiles(gg) * VD_TILE * 8 + 7 * 32 * 4 + 5 * 32 * 8; }
// s_fb bits
#define VF_TOO_CLOSE 1
#define VF_BOUND 2
#define VF_USE_PROF 4
#define VF_HAS_CTRL 8
#define VF_BAD 16   // the length is out of range: a row of NaN
// s_dv rows
#define VF_VCS 0
#define VF_VSTART 1
#define VF_VCTL0 2
#define VF_VCONTROL 3
#define VF_VEND 4

// rows r of the warp: points p in [lo[r], hi[r]] read the per-point friction of their mirror lo[r] + hi[r] - p (tph does
// not flip p_ggv in the backward sweep, DESIGN.md section 7); base: column 0 or 1 of the [n][2] rows
__device__ __forceinline__ void vf_load_mir(double* tile, const double* base, int64_t rs, const int* lo, const int* hi,
                                            int path0, int p0, int lane) {
    const int pt = lane % VD_H, sub = lane / VD_H;
    const int p = p0 + pt;
#pragma unroll 4
    for (int r = sub; r < 32; r += 32 / VD_H) {
        if (p >= lo[r] && p <= hi[r])
            vd_cp_async8(&tile[pt * VD_W + r], base + (size_t)(path0 + r) * rs + 2 * (size_t)(lo[r] + hi[r] - p));
    }
}

// float64 brake chain of the opponent on the race line rolled to `start` (CVPF:166-199): summed el while v > 0.1
__device__ __forceinline__ double vf_opp_stop_dist(const double* __restrict__ G, int M, int start, double v_obj,
                                                   double exp_, double dmq) {
    double v = fmin(v_obj, __ldg(G + 6 * start + 4));
    if (v < 0.0) v = 0.0;   // tph.calc_vel_profile_brake: v_start < 0 -> 0
    double w = v * v, dist = 0.0;
    bool stopped = false;
    for (int i = 0; i < M && v > 0.1; ++i) {
        int r = start + i;
        if (r >= M) r -= M;
        const double e = __ldg(G + 6 * r + 5);
        dist += e;
        if (i < M - 1 && !stopped) {   // kappa has M points, el_lengths M - 1: M - 1 steps
            const double nx = brake_step(w, fabs(__ldg(G + 6 * r + 3)), 14.0, 1.0 / 14.0, exp_, dmq, e);
            if (nx < 0.0) {
                stopped = true;
                v = 0.0;
            } else {
                w = nx;
                v = sqrt(w);
            }
        } else {
            v = 0.0;   // behind the last point the loop ends anyway
        }
    }
    return dist;
}

// EXP1: friction-ellipse exponent 1.0.  GG: per-point friction vf.gg (times gg_scale), else params.gg_ax / gg_ay (times
// gg_scale).  Any length per path (vf.n_pts) and row strides.  Outputs behind a path's end are 0; a path whose length is
// out of [2, n_points] gets a row of NaN and both flags 0.
template <bool EXP1, bool GG>
__global__ void __launch_bounds__(32)
k_velfollow(const __grid_constant__ LtplParams prm, const __grid_constant__ LtplVelFollow vf) {
    extern __shared__ __align__(16) unsigned char vd_smem[];
    double* t_k = reinterpret_cast<double*>(vd_smem);
    double* t_e = t_k + VD_TILE;
    double* t_p = t_e + VD_TILE;   // w pair (control, complete) as one 8-byte element
    double* t_v = t_p + VD_TILE;   // ego brake; vx on the way out
    double* t_gx = t_v + VD_TILE;  // GG: the point's own friction (F1, F2), the complete profile's mirror (B)
    double* t_gy = t_gx + VD_TILE;
    double* t_hx = t_gy + VD_TILE; // GG: the control profile's mirror (B)
    double* t_hy = t_hx + VD_TILE;
    int* s_n = reinterpret_cast<int*>(t_k + vf_tiles(GG) * VD_TILE);
    int* s_o = s_n + 32;
    int* s_z = s_o + 32;   // brake points kept in the vx row
    int* s_lo = s_z + 32;  // control profile [lo, hi]; hi < lo: none
    int* s_hi = s_lo + 32;
    int* s_st = s_hi + 32;  // stop_idx
    int* s_fb = s_st + 32;  // VF_* flag bits
    // Per-lane scalars that the sweeps do not step with live in shared memory, not in registers: the out-of-line pow /
    // division calls of the general-exponent sweeps then have few values to keep across them (no spills)
    double* s_dv = reinterpret_cast<double*>(s_fb + 32);
    __shared__ float s_tab[4 * VR_TAB];
    const int lane = threadIdx.x;
    const int path0 = blockIdx.x * 32;
    const int i = path0 + lane;
    const int n = vf.n_points;
    const bool in = i < vf.n_paths;
    int n_i = in ? n : 0;
    if (in && vf.n_pts) n_i = vf.n_pts[i];
    const bool bad = in && (n_i < 2 || n_i > n);
    if (!in || bad) n_i = 0;
    const bool live = n_i > 0;
    s_n[lane] = n_i;
    s_o[lane] = in ? n : 0;
    vr_stage_axm(prm, s_tab);

    const double v_obj = live ? vf.v_obj[i] : 0.0;
    const double ox = live ? vf.obj_pos[(size_t)i * vf.obj_pos_s] : 0.0;
    const double oy = live ? vf.obj_pos[(size_t)i * vf.obj_pos_s + 1] : 0.0;
    const double dmq = prm.drag_coeff / prm.m_veh;
    const double exp_ = EXP1 ? 1.0 : prm.dyn_model_exp;   // EXP1: no out-of-line pow on the brake chains

    // ---- 0. opponent: nearest race-line point, neighbour rule (get_s_coord closed=True, index [0]), brake chain ----
    const int M = vf.n_glob;
    const double* __restrict__ G = vf.glob_rl;
    const bool staged = (size_t)M * 16 <= (size_t)vf_tiles(GG) * VD_TILE * 8;   // warp uniform
    double2* s_xy = reinterpret_cast<double2*>(vd_smem);
    if (staged) {
        for (int k = lane; k < M; k += 32) s_xy[k] = make_double2(__ldg(G + 6 * k + 1), __ldg(G + 6 * k + 2));
    }
    __syncthreads();
    double bv = LTPL_INF;
    int nb = 0;
    if (staged) {
#pragma unroll 4
        for (int k = 0; k < M; ++k) {   // every lane reads the same point: a broadcast
            const double2 q = s_xy[k];
            const double d = dist2_rn(q.x, q.y, ox, oy);
            if (d < bv) {
                bv = d;
                nb = k;
            }
        }
    } else {
        for (int k0 = 0; k0 < M; k0 += 4) {   // four points in flight
            double qx[4], qy[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int k = min(k0 + u, M - 1);
                qx[u] = __ldg(G + 6 * k + 1);
                qy[u] = __ldg(G + 6 * k + 2);
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const double d = dist2_rn(qx[u], qy[u], ox, oy);
                if (k0 + u < M && d < bv) {
                    bv = d;
                    nb = k0 + u;
                }
            }
        }
    }
    int start = 0;
    double opp_stop_dist = 0.0;
    if (live) {
        const int i1 = (nb == 0) ? M - 1 : nb - 1;   // closed: idx_nb - 1 = -1 is the last point
        const int i2 = (nb + 1 > M - 1) ? 0 : nb + 1;
        const double2 gn = make_double2(__ldg(G + 6 * nb + 1), __ldg(G + 6 * nb + 2));
        const double2 g1 = make_double2(__ldg(G + 6 * i1 + 1), __ldg(G + 6 * i1 + 2));
        const double2 g2 = make_double2(__ldg(G + 6 * i2 + 1), __ldg(G + 6 * i2 + 2));
        start = angle_cmp(gn, ox, oy, g1, g2).ge ? i1 : nb;
        opp_stop_dist = vf_opp_stop_dist(G, M, start, v_obj, exp_, dmq);
    }
    __syncthreads();   // the tile area is free again

    // ---- follow scalars that need no path array (CVPF:139-145, 201-247) ----
    const double safety_in = live ? vf.safety_d[i] : 0.0;
    const double obj_dist = live ? vf.obj_dist[i] : 0.0;
    const double control_d = prm.follow_c_p * safety_in + vf.veh_length;
    const double safety_d = safety_in + vf.veh_length;
    s_fb[lane] = (((obj_dist - safety_d) < 0) ? VF_TOO_CLOSE : 0) | (bad ? VF_BAD : 0);
    const double s_stop = obj_dist - safety_d + opp_stop_dist;
    const double v_ego = live ? vf.v_ego[i] : 0.0;
    double v_control;
    if (prm.follow_control_type == 0) {   // CVPF:28-75
        v_control = v_obj - prm.follow_k_p * (control_d - obj_dist) + prm.follow_k_d * (v_obj - v_ego);
    } else {
        double arg = (control_d - obj_dist) * LTPL_PI / 2 * 1 / prm.follow_tan_w;
        arg = fmin(fmax(arg, -LTPL_PI / 2 + 1e-5), LTPL_PI / 2 - 1e-5);
        v_control = v_obj - tan(arg) * prm.follow_k_p + prm.follow_k_d * (v_obj - v_ego);
    }
    v_control = fmin(fmax(v_control, 0.0), prm.vel_max);
    s_dv[VF_VCONTROL * 32 + lane] = v_control;
    const double v_start = live ? vf.v_start[i] : 0.0;
    const double gs = prm.gg_scale;
    const double inv_ay = 1.0 / (prm.gg_ay * gs);
    const double ax_c = prm.gg_ax * gs;
    const int ntile = (n + VD_H - 1) / VD_H;
    const int n_warp = (int)__reduce_max_sync(LTPL_FULL, (unsigned)n_i);

    // ---- 1. pass F1: s, stop_idx, ego brake profile (CVPF:152-165, 201-209) ----
    const double v0 = fmax(v_start, 0.0);
    double w = v0 * v0, s = 0.0, s_ib = 0.0, s_last = 0.0, v_fl = 0.0, v_st = 0.0;
    int ib = VF_NONE, fl = VF_NONE, stop_idx = VF_NONE, z = n_i;
    bool broke = false;
    for (int tl = 0; tl < ntile; ++tl) {
        const int p0 = tl * VD_H;
        const bool done = !live || p0 >= n_i || (broke && ib != VF_NONE && fl != VF_NONE && stop_idx != VF_NONE);
        if (__all_sync(LTPL_FULL, done)) break;
        vd_load_rows(t_k, vf.kappa, vf.kappa_s, 1, s_n, 0, path0, p0, lane);
        vd_load_rows(t_e, vf.el, vf.el_s, 1, s_n, 1, path0, p0, lane);
        if constexpr (GG) {
            vd_load_rows(t_gx, vf.gg, vf.gg_s, 2, s_n, 0, path0, p0, lane);
            vd_load_rows(t_gy, vf.gg + 1, vf.gg_s, 2, s_n, 0, path0, p0, lane);
        }
        vd_cp_async_wait_all();
        __syncwarp();
#pragma unroll 1
        for (int k = 0; k < VD_H; ++k) {
            const int p = p0 + k;
            if (p < n_i) {
                const double v = (p == 0) ? v0 : (broke ? 0.0 : sqrt(w));
                if (ib == VF_NONE && !(v > 0.1)) {
                    ib = p;
                    s_ib = s;
                }
                if (fl == VF_NONE && v <= v_control) {
                    fl = p;
                    v_fl = v;
                }
                if (stop_idx == VF_NONE && !(s < s_stop)) {
                    stop_idx = p;
                    v_st = v;
                }
                if (p == n_i - 1) {
                    s_last = s;
                    if (stop_idx == VF_NONE) {   // the search stops at the last point
                        stop_idx = p;
                        v_st = v;
                    }
                }
                const double ds = t_e[k * VD_W + lane];
                t_v[k * VD_W + lane] = v;
                if (p < n_i - 1) {
                    if (!broke) {
                        const double kabs = fabs(t_k[k * VD_W + lane]);
                        const double nx = GG ? brake_step(w, kabs, t_gx[k * VD_W + lane] * gs,
                                                          __drcp_rn(t_gy[k * VD_W + lane] * gs), exp_, dmq, ds)
                                             : brake_step(w, kabs, ax_c, inv_ay, exp_, dmq, ds);
                        if (nx < 0.0) {   // negative radicand: standstill, the rest of the profile is 0
                            broke = true;
                            z = p + 1;
                        } else {
                            w = nx;
                        }
                    }
                    s += ds;
                }
            }
        }
        __syncwarp();
        vd_store_rows(t_v, vf.vx, vf.out_s, s_n, path0, p0, lane);
        __syncwarp();
    }

    // ---- follow scalars on the brake profile (CVPF:161-165, 211-292) ----
    double v_end = 0.0, vcs = v_start;
    int idx_c = 0;
    bool use_prof = false, has_ctrl = false, bound = true;
    if (live) {
        const double ego_stop_dist =
            (ib != VF_NONE) ? s_ib : s_last + vf.el[(size_t)i * vf.el_s + n_i - 1];   // el[0:id_brake], el[P-1] included
        if (s_stop > s_last && stop_idx == n_i - 1) {   // v_end from the rolled race line (CVPF:211-223)
            const double s_ends = opp_stop_dist - (s_stop - s_last);
            int idx = 0;
            double s_summed = 0.0;
            while (s_summed < s_ends && idx < M) {
                int r = start + idx;
                if (r >= M) r -= M;
                s_summed += __ldg(G + 6 * r + 5);
                ++idx;
            }
            int r = start + idx;
            while (r >= M) r -= M;
            v_end = __ldg(G + 6 * r + 4);
        }
        if (ego_stop_dist < s_stop) {
            use_prof = true;
            if (v_start > v_control && stop_idx >= 2) {
                // np.argmax(vx_decel <= v_control): 0 for an all-False row; min with stop_idx; 0 -> stop_idx
                idx_c = (fl == VF_NONE) ? 0 : min(fl, stop_idx);
                vcs = (idx_c == fl && fl != VF_NONE) ? v_fl : v_st;
                if (idx_c == 0) {
                    idx_c = stop_idx;
                    vcs = v_st;
                }
            } else {
                if (!(stop_idx >= 2)) bound = false;
                idx_c = 0;
                vcs = v_start;
            }
            has_ctrl = (stop_idx - idx_c) > 0;
        }
    }
    s_z[lane] = min(z, n_i);
    s_lo[lane] = idx_c;
    s_hi[lane] = has_ctrl ? stop_idx : -1;
    s_st[lane] = stop_idx;
    s_fb[lane] |= (bound ? VF_BOUND : 0) | (use_prof ? VF_USE_PROF : 0) | (has_ctrl ? VF_HAS_CTRL : 0);
    s_dv[VF_VCS * 32 + lane] = vcs;
    s_dv[VF_VSTART * 32 + lane] = v_start;
    s_dv[VF_VCTL0 * 32 + lane] = vcs;   // vx_control[0] until pass B has it
    s_dv[VF_VEND * 32 + lane] = v_end;
    __syncwarp();

    // ---- 2. pass F2: complete profile on [0, n - 1] (CVPF:297-310, no v_end) and control profile on [idx_c, stop_idx]
    //      (CVPF:263-276) forward; the w pair of a point leaves as one 8-byte element of the ax row ----
    const VRCfg c = vr_make_cfg(prm, s_tab);
    const float wmax = (float)(prm.vel_max * prm.vel_max);
    const float wcap = (float)(v0 * v0);
    double* scr = vf.ax;   // the caller's ax rows: (w control, w complete) pairs
    {
        VRSweep f, g;
        f.start(0.0f, 0.0f, 0.0f);
        g.start(0.0f, 0.0f, 0.0f);
        VRSeg seg, seg_c;
        seg.load(c, 1);
        seg_c.load(c, 1);
        float e_prev = 0.0f;
        for (int tl = 0; tl < ntile; ++tl) {
            const int p0 = tl * VD_H;
            if (p0 >= n_warp) break;
            vd_load_rows(t_k, vf.kappa, vf.kappa_s, 1, s_n, 0, path0, p0, lane);
            vd_load_rows(t_e, vf.el, vf.el_s, 1, s_n, 1, path0, p0, lane);
            if constexpr (GG) {
                vd_load_rows(t_gx, vf.gg, vf.gg_s, 2, s_n, 0, path0, p0, lane);
                vd_load_rows(t_gy, vf.gg + 1, vf.gg_s, 2, s_n, 0, path0, p0, lane);
            }
            vd_cp_async_wait_all();
            __syncwarp();
#pragma unroll 1
            for (int k = 0; k < VD_H; ++k) {
                const int p = p0 + k;
                const bool on = p < n_i;
                const double iay = GG ? __drcp_rn(t_gy[k * VD_W + lane] * gs) : inv_ay;
                const float axq = GG ? (float)(t_gx[k * VD_W + lane] * gs) : c.ax_max;
                const float kq = (float)(fabs(t_k[k * VD_W + lane]) * iay);
                const float e2 = (float)(2.0 * t_e[k * VD_W + lane]);
                float wf, wc = 0.0f;
                if (p == 0) {
                    wf = vr_w_start(kq, wmax, wcap);
                    f.start(wf, kq, axq);
                } else {
                    wf = f.fwd<EXP1>(c, seg, kq, axq, e_prev, wmax, live && on);
                }
                // control: every lane steps (the machine-limit lookup votes across the warp), a lane outside its range
                // without using the result; at lo its sweep starts afresh
                const int lo = s_lo[lane], hi = s_hi[lane];
                const double vcl = s_dv[VF_VCONTROL * 32 + lane];
                const float wmax_c = (float)(vcl * vcl);
                wc = g.fwd<EXP1>(c, seg_c, kq, axq, e_prev, wmax_c, p > lo && p <= hi);
                if (p == lo) {
                    const double vcs_p = fmax(s_dv[VF_VCS * 32 + lane], 0.0);
                    g = VRSweep();
                    wc = vr_w_start(kq, wmax_c, (float)(vcs_p * vcs_p));
                    g.start(wc, kq, axq);
                }
                if (p == hi) {
                    const double ve_p = fmax(s_dv[VF_VEND * 32 + lane], 0.0);
                    vr_clamp_end(wc, (float)(ve_p * ve_p));
                }
                e_prev = e2;
                if (on)   // low word: control, high word: complete (float index 2p, 2p + 1 of the ax row)
                    t_k[k * VD_W + lane] = __hiloint2double(__float_as_int(wf), __float_as_int(wc));
            }
            __syncwarp();
            vd_store_rows(t_k, scr, vf.out_s, s_n, path0, p0, lane);
            __syncwarp();
        }
    }

    // ---- 3. pass B: both backward sweeps, merge (CVPF:278-292, 311), vx, ax, flags; zeros behind the end ----
    VRSweep b, h;
    double v_next = 0.0;
    for (int tl = ntile - 1; tl >= 0; --tl) {
        const int p0 = tl * VD_H;
        vd_load_rows(t_k, vf.kappa, vf.kappa_s, 1, s_n, 0, path0, p0, lane);
        vd_load_rows(t_e, vf.el, vf.el_s, 1, s_n, 1, path0, p0, lane);
        vd_load_rows(t_p, scr, vf.out_s, 1, s_n, 0, path0, p0, lane);
        vd_load_rows(t_v, vf.vx, vf.out_s, 1, s_z, 0, path0, p0, lane);
        if constexpr (GG) {
            vd_load_rows<true>(t_gx, vf.gg, vf.gg_s, 2, s_n, 0, path0, p0, lane);
            vd_load_rows<true>(t_gy, vf.gg + 1, vf.gg_s, 2, s_n, 0, path0, p0, lane);
            vf_load_mir(t_hx, vf.gg, vf.gg_s, s_lo, s_hi, path0, p0, lane);
            vf_load_mir(t_hy, vf.gg + 1, vf.gg_s, s_lo, s_hi, path0, p0, lane);
        }
        vd_cp_async_wait_all();
        __syncwarp();
#pragma unroll 1
        for (int k = VD_H - 1; k >= 0; --k) {
            const int p = p0 + k;
            if (p >= n) continue;   // warp uniform
            double vx = 0.0, ax = 0.0;
            const int n_i = s_n[lane];   // (shared memory: one value less across the sweeps' calls)
            if (p < n_i) {
                const double kabs = fabs(t_k[k * VD_W + lane]);
                const float e2 = (float)(2.0 * t_e[k * VD_W + lane]);
                const double iay = GG ? __drcp_rn(t_gy[k * VD_W + lane] * gs) : inv_ay;
                const float axq = GG ? (float)(t_gx[k * VD_W + lane] * gs) : c.ax_max;
                const float kq = (float)(kabs * iay);
                const double pd = t_p[k * VD_W + lane];
                const float2 pr = make_float2(__int_as_float(__double2loint(pd)), __int_as_float(__double2hiint(pd)));
                float wf = pr.y;
                if (p < n_i - 1)
                    wf = b.bwd<EXP1>(c, pr.y, kq, axq, e2, wmax);
                else
                    b.start(pr.y, kq, axq);
                const double v_cmp = (double)vr_sqrt(wf);
                double prof;
                const int fb = s_fb[lane], lo = s_lo[lane];
                if (!(fb & VF_USE_PROF)) {
                    prof = (p < s_z[lane]) ? t_v[k * VD_W + lane] : 0.0;   // ego brake profile (CVPF:293-294)
                } else if (p < lo) {
                    prof = t_v[k * VD_W + lane];                   // vx_decel[:-1]
                } else if (p <= s_st[lane]) {
                    if (fb & VF_HAS_CTRL) {
                        const double vcl = s_dv[VF_VCONTROL * 32 + lane];
                        const double iay_c = GG ? __drcp_rn(t_hy[k * VD_W + lane] * gs) : inv_ay;
                        const float axq_c = GG ? (float)(t_hx[k * VD_W + lane] * gs) : c.ax_max;
                        const float kq_c = (float)(kabs * iay_c);
                        float wc = pr.x;
                        if (p < s_hi[lane])
                            wc = h.bwd<EXP1>(c, pr.x, kq_c, axq_c, e2, (float)(vcl * vcl));
                        else
                            h.start(pr.x, kq_c, axq_c);
                        prof = (double)vr_sqrt(wc);
                        if (p == lo) s_dv[VF_VCTL0 * 32 + lane] = sqrt((double)wc);
                    } else {
                        prof = s_dv[VF_VCS * 32 + lane];           // vx_control = [vx_control_start]
                    }
                } else {
                    prof = 0.0;
                }
                vx = (prof < v_cmp) ? prof : v_cmp;
                if (p < n_i - 1) ax = (v_next * v_next - vx * vx) * fast_rcp(2.0 * t_e[k * VD_W + lane]);
                v_next = vx;
            } else if (s_fb[lane] & VF_BAD) {
                vx = ax = CUDART_NAN;
            }
            t_v[k * VD_W + lane] = vx;
            t_k[k * VD_W + lane] = ax;
        }
        __syncwarp();
        vd_store_rows(t_v, vf.vx, vf.out_s, s_o, path0, p0, lane);
        vd_store_rows(t_k, vf.ax, vf.out_s, s_o, path0, p0, lane);
        __syncwarp();
    }

    __syncwarp();
    if (in) {
        const int fb = s_fb[lane];
        bool bound = (fb & VF_BOUND) != 0;
        if (fb & VF_USE_PROF) {   // CVPF:276-278, 290-291
            const double vcs = s_dv[VF_VCS * 32 + lane], v_ctl0 = s_dv[VF_VCTL0 * 32 + lane];
            const double v_st = s_dv[VF_VSTART * 32 + lane];
            if ((fb & VF_HAS_CTRL) && fabs(v_ctl0 - vcs) > 1.0) bound = false;
            const double prof0 = (s_lo[lane] > 0) ? fmax(v_st, 0.0) : v_ctl0;
            if (fabs(prof0 - v_st) > 1.0) bound = false;
        }
        vf.too_close[i] = (live && (fb & VF_TOO_CLOSE)) ? 1 : 0;
        vf.vel_bound[i] = (live && bound) ? 1 : 0;
    }
}
