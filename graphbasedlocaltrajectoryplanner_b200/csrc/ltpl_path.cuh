// ltpl_path.cuh -- k_path: edge -> path assembly (MOPG:259-297), C2 spline refit (tph.calc_splines as a tridiagonal
// system in the knot tangents, MOPG:305-309), re-evaluation x, y, psi, kappa at the per-edge sample counts
// (tph.interp_splines(stepnum_fixed) + calc_head_curv_an, MOPG:312-322) and stitching with the constant segment
// (OTH:433-472).  One WARP per (action slot, scenario).
#pragma once
#include "ltpl_plan.cuh"

__host__ __device__ inline size_t path_smem_bytes_per_warp(int h_max) {
    // doubles: px, py, el, mx, my, cp, dx, dy + five more rows of the tridiagonal solve (h_max each) ;
    // ints: nidx, eid, nsamp, soff (h_max each)
    size_t s = sizeof(double) * 13 * (size_t)h_max + sizeof(int) * 4 * (size_t)h_max;
    return (s + 15) & ~(size_t)15;
}

// append path q to the dense work queue of its class (0: follow, 1: straight / left / right) for k_vel
__device__ __forceinline__ void enqueue_path(const LtplBuffers& bf, const LtplDims& dm, int q) {
    const int nq = LTPL_NSLOT * dm.sub_cnt;   // the window's own [2][nq] part of the queue buffer
    const int cls = (bf.action_id[q] == LTPL_ACT_FOLLOW) ? 0 : 1;
    const int pos = atomicAdd(&bf.queue_cnt[4 + 4 * dm.sub_id + cls], 1);
    if (pos < nq) bf.queue[2 * LTPL_NSLOT * dm.sub_off + cls * nq + pos] = q;
    atomicAdd(&bf.queue_cnt[cls], 1);         // totals over all windows (statistics)
}

#ifndef LTPL_PATH_MINB
#define LTPL_PATH_MINB 8
#endif
// STATE: stateful tick (ltpl_state.cuh): the constant part and the list prefixes come from the previous tick's buffers,
// except for a scenario restarted in this tick (LTPL_STATE_RESTARTED): set_startpos's, as in a first tick (const_view)
template <bool STATE>
__global__ void __launch_bounds__(LTPL_WARPS_PER_CTA * 32, LTPL_PATH_MINB)
k_path(const __grid_constant__ LatDev lt, const __grid_constant__ LtplParams prm,
       const __grid_constant__ LtplDims dm, const __grid_constant__ LtplBuffers bf) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31;
    const int wib = threadIdx.x >> 5;
    const int B = dm.batch;
    const int q = sub_path(dm, LTPL_WARPS_PER_CTA);
    if (q < 0) return;
    const int b = q % B;
    const int st = bf.status[q];
    if (!(st & LTPL_ST_FOUND)) return;
    const int H = dm.h_max;
    unsigned char* base = smem_raw + path_smem_bytes_per_warp(H) * wib;
    double* kx = reinterpret_cast<double*>(base);
    double* ky = kx + H;
    double* kel = ky + H;
    double* mx = kel + H;
    double* my = mx + H;
    double* cp = my + H;
    double* dxp = cp + H;
    double* dyp = dxp + H;
    double* pcr = dyp + H;   // [5][H]
    int* nidx = reinterpret_cast<int*>(pcr + 5 * H);
    int* eid = nidx + H;
    int* nsamp = eid + H;
    int* soff = nsamp + H;   // first sample of every edge

    const int p0 = bf.const_len[b];
    const size_t pplane = (size_t)LTPL_NSLOT * B * dm.p_max;
    const ConstView cv = const_view<STATE>(dm, bf, b, B);
    const bool mem = STATE && cv.mem;   // a constant in k_path<false>: its code is that of a kernel without memory
    const double* cs = cv.seg;
    const size_t cplane = cv.plane;
    const int cnd = mem ? bf.st_info[b].const_nodes : 1;   // list entries in front of the start node
    double* pp = bf.path + (size_t)q * dm.p_max;
    int* node_idx = bf.node_idx + (size_t)q * H;
    double* coeff = bf.coeff + (size_t)q * H * 8;

    const int n_nodes = bf.n_nodes[q];  // incl. the leading (-1, -1)
    const int nseg = n_nodes - 1 - cnd; // segments of the new plan

    if (st & LTPL_ST_CONST_ONLY) {  // OTH:481-506: constant segment incl. its last point
        for (int k = lane; k < p0; k += 32)
            for (int c = 0; c < 5; ++c) pp[c * pplane + k] = cs[c * cplane + k];
        if (lane == 0) {
            if (mem) {   // OTH:486-501: memory lists up to and including the start node
                for (int i = 0; i < cnd; ++i) node_idx[i] = cv.node_idx[i] - cv.m;
                for (int i = 0; i < min(cnd + 1, cv.rows) * 8; ++i) coeff[i] = cv.coeff[i];
            } else {
                node_idx[0] = 0;
                for (int c = 0; c < 8; ++c) coeff[c] = bf.const_coeff[(size_t)b * 8 + c];
            }
            node_idx[cnd] = p0 - 1;
            bf.path_len[q] = p0;
            enqueue_path(bf, dm, q);
        }
        return;
    }

    // ---- segment bookkeeping (MOPG:268-297) ----
    const int* es = bf.edge_seq + (size_t)q * H;
    for (int i = lane; i < nseg; i += 32) {
        const int e = es[i];
        const int so0 = lt.samp_off[e], so1 = lt.samp_off[e + 1];
        eid[i] = e;
        soff[i] = so0;
        nsamp[i] = so1 - so0;
        kel[i] = lt.edge_len[e];
        const double2 p = lt.samp_xy[so0];
        kx[i] = p.x;
        ky[i] = p.y;
        if (i == nseg - 1) {
            const double2 pl = lt.samp_xy[so1 - 1];
            kx[nseg] = pl.x;
            ky[nseg] = pl.y;
        }
    }
    __syncwarp();
    {   // exclusive prefix sum of (n_i - 1): index of every node in the fused sample array (warp scan, 32 segments a round)
        int carry = 0;
        #pragma unroll 1
        for (int i0 = 0; i0 < nseg; i0 += 32) {
            const int i = i0 + lane;
            const int v = (i < nseg) ? nsamp[i] - 1 : 0;
            int inc = v;
#pragma unroll
            for (int off = 1; off < 32; off <<= 1) {
                const int up = __shfl_up_sync(LTPL_FULL, inc, off);
                if (lane >= off) inc += up;
            }
            if (i < nseg) nidx[i] = carry + inc - v;
            carry += __shfl_sync(LTPL_FULL, inc, 31);
        }
        if (lane == 0) nidx[nseg] = carry;  // last node sits on the last sample
    }
    __syncwarp();
    const int p_new = nidx[nseg] + 1;
    // closest_path_index(start node) on the constant segment == its last point (OTH:398-404); stateful tick without a
    // constant segment (p0 == 0, OTH:405-411): nothing in front of the new path
    const int loc = (STATE && p0 == 0) ? 0 : p0 - 1;
    const int p_tot = loc + p_new;
    if (p_tot > dm.p_max) {
        if (lane == 0) {
            bf.status[q] = st & ~LTPL_ST_FOUND;
            bf.action_id[q] = LTPL_ACT_NONE;
            atomicOr(&bf.sc_flags[b], LTPL_SC_CAPACITY);
        }
        return;
    }

    // ---- C2 spline through the nodes: tridiagonal system in the knot tangents m_k (== tph.calc_splines) ----
    // MOPG:300-303: heading at the end of the constant segment, else of the first sample of the first edge
    const double psi_s = (STATE && p0 == 0) ? lt.edge_psi0[eid[0]] : cs[2 * cplane + p0 - 1];
    const double psi_e = lt.edge_psi1[eid[nseg - 1]];       // MOPG:307: psi of the last sample
    // rows k = 1 .. nseg-1:  (2/el[k-1]) m[k-1] + 4 (1/el[k-1] + 1/el[k]) m[k] + (2/el[k]) m[k+1] = r[k]
    // solved by PARALLEL CYCLIC REDUCTION: every row eliminates its two neighbours at distance s = 1, 2, 4, ...; after
    // ceil(log2(n)) rounds the rows are decoupled.  All lanes work in every round (a Thomas sweep is n dependent steps on
    // one lane per right-hand side); the system is strictly diagonally dominant (4 : 1 : 1), so the reduction is as stable
    // as the elimination (agreement with tph's dense LAPACK solve <= 1e-13, tests compare the coefficients at 1e-6).
    // tangents (cos, sin)(psi + pi / 2) = (-sin psi, cos psi): one sincos per heading
    double sn_s, cs_s, sn_e, cs_e;
    sincos(psi_s, &sn_s, &cs_s);
    sincos(psi_e, &sn_e, &cs_e);
    const double m0x = -sn_s, m0y = cs_s, mex = -sn_e, mey = cs_e;
    const int n = nseg - 1;
    // two sets of rows (a, b, c, x, y) used alternately (set 1 borrows mx / my for its right-hand sides); the tangents
    // are written to mx / my at the end
    double* A0 = cp;
    double* B0 = dxp;
    double* C0 = dyp;
    double* X0 = pcr;
    double* Y0 = pcr + H;
    double* A1 = pcr + 2 * H;
    double* B1 = pcr + 3 * H;
    double* C1 = pcr + 4 * H;
    double* X1 = mx;
    double* Y1 = my;
    for (int k = 1 + lane; k < nseg; k += 32) {
        const double i0 = fast_rcp(kel[k - 1]), i1 = fast_rcp(kel[k]);
        const double lo = 2.0 * i0, up = 2.0 * i1;
        double rx = 6.0 * ((kx[k] - kx[k - 1]) * (i0 * i0) + (kx[k + 1] - kx[k]) * (i1 * i1));
        double ry = 6.0 * ((ky[k] - ky[k - 1]) * (i0 * i0) + (ky[k + 1] - ky[k]) * (i1 * i1));
        if (k == 1) {
            rx -= lo * m0x;
            ry -= lo * m0y;
        }
        if (k == nseg - 1) {
            rx -= up * mex;
            ry -= up * mey;
        }
        A0[k] = (k == 1) ? 0.0 : lo;
        B0[k] = 2.0 * (lo + up);
        C0[k] = (k == nseg - 1) ? 0.0 : up;
        X0[k] = rx;
        Y0[k] = ry;
    }
    __syncwarp();
    #pragma unroll 1
    for (int sd = 1; sd < n; sd <<= 1) {
        for (int k = 1 + lane; k <= n; k += 32) {
            double a = 0.0, c = 0.0, bb = B0[k], x = X0[k], y = Y0[k];
            if (k - sd >= 1) {
                const double al = -A0[k] * fast_rcp(B0[k - sd]);
                a = al * A0[k - sd];
                bb += al * C0[k - sd];
                x += al * X0[k - sd];
                y += al * Y0[k - sd];
            }
            if (k + sd <= n) {
                const double ga = -C0[k] * fast_rcp(B0[k + sd]);
                c = ga * C0[k + sd];
                bb += ga * A0[k + sd];
                x += ga * X0[k + sd];
                y += ga * Y0[k + sd];
            }
            A1[k] = a;
            B1[k] = bb;
            C1[k] = c;
            X1[k] = x;
            Y1[k] = y;
        }
        __syncwarp();
        double* t;
        t = A0; A0 = A1; A1 = t;
        t = B0; B0 = B1; B1 = t;
        t = C0; C0 = C1; C1 = t;
        t = X0; X0 = X1; X1 = t;
        t = Y0; Y0 = Y1; Y1 = t;
    }
    for (int k = 1 + lane; k <= n; k += 32) {
        const double inv = fast_rcp(B0[k]);
        const double vx = X0[k] * inv, vy = Y0[k] * inv;
        mx[k] = vx;
        my[k] = vy;
    }
    if (lane == 0) {
        mx[0] = m0x;
        my[0] = m0y;
        mx[nseg] = mex;
        my[nseg] = mey;
    }
    __syncwarp();

    // ---- stitched bookkeeping (OTH:458-472) ----
    for (int i = lane; i <= nseg; i += 32) node_idx[cnd + i] = nidx[i] + loc;
    if (mem) {
        for (int i = lane; i < cnd; i += 32) node_idx[i] = cv.node_idx[i] - cv.m;
        for (int i = lane; i < cnd * 8; i += 32) coeff[i] = cv.coeff[i];
    }
    if (!mem && lane < 8) coeff[lane] = bf.const_coeff[(size_t)b * 8 + lane];
    if (lane == 0) {
        if (!mem) node_idx[0] = 0;
        bf.path_len[q] = p_tot;
        enqueue_path(bf, dm, q);
    }
    for (int i = lane; i < nseg; i += 32) {
        const double e0 = kel[i];
        const double dx = kx[i + 1] - kx[i], dy = ky[i + 1] - ky[i];
        const double a1x = e0 * mx[i], e1x = e0 * mx[i + 1];
        const double a1y = e0 * my[i], e1y = e0 * my[i + 1];
        double* c = coeff + (size_t)(cnd + i) * 8;
        c[0] = kx[i]; c[1] = a1x; c[2] = 3 * dx - 2 * a1x - e1x; c[3] = -2 * dx + a1x + e1x;
        c[4] = ky[i]; c[5] = a1y; c[6] = 3 * dy - 2 * a1y - e1y; c[7] = -2 * dy + a1y + e1y;
    }
    // constant part (OTH:442-444): everything but the last point of the constant segment
    for (int k = lane; k < loc; k += 32) {   // (five loads in flight, then five stores)
        const double v0 = cs[k], v1 = cs[cplane + k], v2 = cs[2 * cplane + k], v3 = cs[3 * cplane + k], v4 = cs[4 * cplane + k];
        pp[k] = v0;
        pp[pplane + k] = v1;
        pp[2 * pplane + k] = v2;
        pp[3 * pplane + k] = v3;
        pp[4 * pplane + k] = v4;
    }
    __syncwarp();

    // ---- re-evaluation at the per-edge sample counts (MOPG:312-322); el column keeps the offline chords (q2) ----
    for (int p = lane; p < p_new; p += 32) {
        int lo_i = 0, hi_i = nseg - 1;  // largest i with nidx[i] <= p (the very last point belongs to the last segment)
        while (lo_i < hi_i) {
            const int mid = (lo_i + hi_i + 1) >> 1;
            if (nidx[mid] <= p)
                lo_i = mid;
            else
                hi_i = mid - 1;
        }
        const int i = lo_i;
        const int k = p - nidx[i];
        const int n_i = nsamp[i];
        const double el_off = lt.samp_el[soff[i] + k];   // (issued before the arithmetic that hides its latency)
        const double e0 = kel[i];
        const double dx = kx[i + 1] - kx[i], dy = ky[i + 1] - ky[i];
        const double a0x = kx[i], a1x = e0 * mx[i], e1x = e0 * mx[i + 1];
        const double a0y = ky[i], a1y = e0 * my[i], e1y = e0 * my[i + 1];
        const double a2x = 3 * dx - 2 * a1x - e1x, a3x = -2 * dx + a1x + e1x;
        const double a2y = 3 * dy - 2 * a1y - e1y, a3y = -2 * dy + a1y + e1y;
        double t, x, y;
        if (p == p_new - 1) {  // incl_last_point: coordinates = sum of the coefficients, t = 1
            t = 1.0;
            x = ((a0x + a1x) + a2x) + a3x;
            y = ((a0y + a1y) + a2y) + a3y;
        } else {
            t = k * fast_rcp((double)(n_i - 1));  // np.linspace(0, 1, n_i)[k] (2e-16 relative)
            x = cubic_rn(a0x, a1x, a2x, a3x, t);
            y = cubic_rn(a0y, a1y, a2y, a3y, t);
        }
        double psi, kap;
        head_curv(a1x, a2x, a3x, a1y, a2y, a3y, t, &psi, &kap);
        const int o = loc + p;
        pp[0 * pplane + o] = x;
        pp[1 * pplane + o] = y;
        pp[2 * pplane + o] = psi;
        pp[3 * pplane + o] = kap;
        pp[4 * pplane + o] = el_off;
    }
}
