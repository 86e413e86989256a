// ltpl_pathcoord.cuh -- positions on the caller's polylines (sm_90a): get_s_coord, closest_path_index and
// check_inside_bounds of the reference for N queries per launch (ltpl_path_coord_batch).
//
// One warp per query.  The nearest point is the tick's scan (closest_point_scan, first minimum), the neighbour choice
// angle_cmp with its exact atan2 fallback, the foot of the perpendicular foot_ds and the bound test inside_from_pair's
// linspace emulation: the helpers the tick's golden vectors pin, here behind a strided gather instead of a lattice array.
#pragma once
#include "ltpl_common.cuh"

#define PC_WARPS 8   // queries per CTA

// point j of one row: x[j * ps], y[j * ps]
struct PcLine {
    const double* x;
    const double* y;
    int64_t ps;
    __device__ __forceinline__ double2 operator()(int j) const { return make_double2(x[j * ps], y[j * ps]); }
};
// check_inside_bounds.py:28: the centre line (bound1 + bound2) / 2
struct PcCenter {
    PcLine b1, b2;
    __device__ __forceinline__ double2 operator()(int j) const {
        const double2 u = b1(j), w = b2(j);
        return make_double2(__ddiv_rn(__dadd_rn(u.x, w.x), 2.0), __ddiv_rn(__dadd_rn(u.y, w.y), 2.0));
    }
};

// element k of get_s_coord's s_array after the leading-zero insertion (get_s_coord.py:62-68), k = -1 reading the last
// one, s_array = np.cumsum of the chord lengths (get_s_coord.py:64): the first chords summed in index order, as
// np.cumsum does -- the lanes compute 32 chords at a time, every lane adds them one by one.  NaN where the reference
// raises the IndexError (no insertion and k = n - 1: the cumulated array has n - 1 elements).  Warp-collective.
__device__ __forceinline__ double chord_s(const PcLine& L, int n, int k, int lane) {
    const double2 p0 = L(0), p1 = L(1);
    const bool ins = sqrt(dist2_rn(p1.x, p1.y, p0.x, p0.y)) > 0.05;
    if (!ins && k == n - 1) return CUDART_NAN;
    const int j = (k < 0) ? n - 1 : (ins ? k : k + 1);   // chords 0 .. j - 1
    double acc = 0.0;
    #pragma unroll 1
    for (int i0 = 0; i0 < j; i0 += 32) {
        double c = 0.0;
        if (i0 + lane < j) {
            const double2 a = L(i0 + lane), b = L(i0 + lane + 1);
            c = sqrt(dist2_rn(b.x, b.y, a.x, a.y));   // np.diff, np.power, np.sum(axis=1), np.sqrt
        }
#pragma unroll
        for (int l = 0; l < 32; ++l) {
            const double v = __shfl_sync(LTPL_FULL, c, l);
            if (i0 + l < j) acc = __dadd_rn(acc, v);
        }
    }
    return acc;
}

// element k of a given s_array row (n elements, element stride es) after the insertion, k = -1 reading the last one
__device__ __forceinline__ double given_s(const double* sa, int64_t es, int n, int k) {
    if (k < 0) return sa[(n - 1) * es];
    if (sa[0] > 0.05) return k == 0 ? 0.0 : sa[(k - 1) * es];
    return sa[k * es];
}

template <int MODE>
__global__ void __launch_bounds__(PC_WARPS * 32) k_pathcoord(const __grid_constant__ LtplPathCoord pc) {
    const int64_t q = (int64_t)blockIdx.x * PC_WARPS + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (q >= pc.n_queries) return;
    const int n = pc.n_pts ? pc.n_pts[q] : pc.m_points;
    const double px = pc.pos[q * pc.pos_s[0]], py = pc.pos[q * pc.pos_s[0] + pc.pos_s[1]];
    const PcLine L = {pc.x + q * pc.line_s, pc.y + q * pc.line_s, pc.pt_s};
    bool ok = n >= 2 && n <= pc.m_points && isfinite(px) && isfinite(py);
    int nb = 0;
    if (ok) {
        if (MODE == LTPL_PC_INSIDE_BOUNDS) {
            const PcCenter C = {L, {pc.x2 + q * pc.line2_s, pc.y2 + q * pc.line2_s, pc.pt2_s}};
            nb = closest_point_scan(C, n, px, py, lane).i;
        } else {
            nb = closest_point_scan(L, n, px, py, lane).i;
        }
        ok = nb < n;   // a row without a point at a finite distance
    }
    if (MODE == LTPL_PC_CLOSEST) {
        if (lane == 0) pc.idx[q] = ok ? nb : -1;
        return;
    }
    if (!ok) {
        if (lane == 0) {
            if (MODE == LTPL_PC_INSIDE_BOUNDS) {
                pc.inside[q] = -1;
            } else {
                if (pc.s) pc.s[q] = CUDART_NAN;
                pc.closest[2 * q] = pc.closest[2 * q + 1] = -2;
            }
        }
        return;
    }
    // get_s_coord.py:38-58: neighbours (NumPy's -1 kept for a closed line), the side of the larger angle
    const bool closed = MODE == LTPL_PC_INSIDE_BOUNDS || pc.closed;
    int idx1, idx2;
    if (closed) {
        idx1 = nb - 1;
        idx2 = (nb + 1 > n - 1) ? 0 : nb + 1;
    } else {
        idx1 = max(nb - 1, 0);
        idx2 = min(nb + 1, n - 1);
    }
    const int a1 = (idx1 < 0) ? n - 1 : idx1;
    if (MODE == LTPL_PC_INSIDE_BOUNDS) {
        const PcLine B2 = {pc.x2 + q * pc.line2_s, pc.y2 + q * pc.line2_s, pc.pt2_s};
        const PcCenter C = {L, B2};
        const bool ge = angle_cmp(C(nb), px, py, C(a1), C(idx2)).ge;
        const int i0 = ge ? a1 : nb, i1 = ge ? nb : idx2;
        const bool in = inside_from_pair(C(i0), C(i1), L, B2, i0, i1, px, py, lane);
        if (lane == 0) pc.inside[q] = in ? 1 : 0;
        return;
    }
    const double2 pn = L(nb), p1 = L(a1), p2 = L(idx2);
    const AngCmp c = angle_cmp(pn, px, py, p1, p2);
    if (MODE == LTPL_PC_S_COORD) {
        // get_s_coord.py:54-90
        const int k = c.gt ? idx1 : nb;
        const double ds = c.gt ? foot_ds(p1, pn, px, py) : foot_ds(pn, p2, px, py);
        double sb;
        if (pc.s_array) {
            sb = given_s(pc.s_array + q * pc.s_array_s, pc.s_array_es, n, k);
        } else {
            sb = chord_s(L, n, k, lane);
        }
        if (lane == 0) pc.s[q] = __dadd_rn(sb, ds);
    } else if (lane == 0 && pc.s) {
        pc.s[q] = CUDART_NAN;   // only_index: the reference returns None
    }
    if (lane == 0) {   // get_s_coord.py:94-97
        pc.closest[2 * q] = c.ge ? idx1 : nb;
        pc.closest[2 * q + 1] = c.ge ? nb : idx2;
    }
}
