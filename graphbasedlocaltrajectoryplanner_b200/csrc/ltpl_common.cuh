// ltpl_common.cuh -- device-side lattice view + numerics helpers shared by all kernels (sm_90a).
//
// Numerics contract (DESIGN.md "Numerics"): every DECISION of the reference path (nearest-index argmins, collision
// tests, interval tests on s-coordinates, DP relax / argmin) is taken in IEEE float64 with the same operation order as
// NumPy executes it (this translation unit is compiled with -fmad=false, and the helpers below additionally use
// explicit round-to-nearest intrinsics so that a later relaxation of the flag cannot change decisions).
#pragma once
#include <cuda_runtime.h>
#include <math_constants.h>
#include <stdint.h>

#include "ltpl_b200.h"

// optional phase timing (debug builds only: -DLTPL_PROFILE_PHASES): cycles per phase summed over lane 0 of every warp
// (slots 0..15: velocity kernels, 16..31: k_plan)
#ifdef LTPL_PROFILE_PHASES
__device__ unsigned long long g_phase[32];
#define LTPL_PH_INIT long long _t0 = clock64();
#define LTPL_PH(k)                                                                                   \
    {                                                                                                \
        long long _t1 = clock64();                                                                   \
        if ((threadIdx.x & 31) == 0) atomicAdd(&g_phase[k], (unsigned long long)(_t1 - _t0));        \
        _t0 = clock64();                                                                             \
    }
#else
#define LTPL_PH_INIT
#define LTPL_PH(k)
#endif

#define LTPL_FULL 0xffffffffu
#define LTPL_PI 3.141592653589793
#define LTPL_INF CUDART_INF

// resolved device pointers of the lattice blob
struct LatDev {
    int L, Nn, E, S, n_glob, closed, plan_mode, max_nodes, max_window_edges;
    double lat_offset, lat_res, step, vel_decrease_lat, veh_width, veh_length, virt_cost, min_plan_horizon;
    const int* node_off;
    const int* rl_idx;
    const double* s_rl;
    const double* vel_rl;
    const double2* refline;
    const double2* raceline;
    const double2* bound1;
    const double2* bound2;
    const double2* center;
    const double2* node_xy;
    const double* node_psi;
    const int* node_layer;
    const int2* in_off;
    const int* edge_layer_off;
    const int* edge_src;
    const int* edge_dst;
    const double* edge_cost;
    const double* edge_len;
    const double* edge_psi1;
    const double* edge_psi0;
    const int* samp_off;
    const double2* samp_xy;
    const double* samp_el;
    const int* samp_edge;
    const double* glob_rl;  // [n_glob - 1][6]
    const double2* glob_xy; // [n_glob - 1]
    const LtplEdgeRec* edge_rec;   // [E] (cost, src, dst) of every edge in one 16-byte record (DP inner loop)
    const int* tab_reach;          // [Nn] follow table (k_follow_table): steps | tie << 8
    const unsigned char* tab_node; // [Nn][tab_stride] node index per step
    const int* tab_edge;           // [Nn][tab_stride] edge id per step
    int tab_stride;
    // nearest-vertex grids (lattice_blob.nearest_grid): cell -> (first << 6 | count) candidates that contain the nearest
    // vertex of every position inside the cell
    const int* grid_center;
    const int* grid_refline;
    const int* grid_raceline;
    const int* grid_glob;
    int grid_nx, grid_ny, grid_cyclic;
    double grid_x0, grid_y0, grid_inv_cell;
};

#ifndef LTPL_DEFAULT_SUB
#define LTPL_DEFAULT_SUB 4     // scenario windows per tick
#endif
#ifndef LTPL_SUB_MIN
#define LTPL_SUB_MIN 512       // ... but no window below this many scenarios unless ltpl_set_subbatches asks for it
#endif
struct LtplLattice {
    LtplLatticeHeader h;
    LatDev d;
    // a tick runs as n_sub scenario windows: window 0 on the caller's stream, window s > 0 on aux[s - 1], forked from and
    // joined into the caller's stream with events (ltpl_set_subbatches)
    int n_sub = 1, sub_min = LTPL_SUB_MIN;
    cudaStream_t aux[LTPL_MAX_SUB - 1] = {};
    cudaEvent_t ev_fork = nullptr, ev_join[LTPL_MAX_SUB - 1] = {};
    // dynamic shared memory each kernel family (ltpl_api.cu: SmemFamily) may use on this handle's device
    mutable size_t smem_allowed[4] = {};
    mutable int plan_carveout = -1;   // k_plan's preferred shared-memory carveout last set by this handle (percent)
};

// scenario of a one-warp-per-scenario kernel inside the launch's sub-batch window (-1: none)
__device__ __forceinline__ int sub_scenario(const LtplDims& dm, int warps_per_cta) {
    const int i = blockIdx.x * warps_per_cta + (threadIdx.x >> 5);
    return (i < dm.sub_cnt) ? dm.sub_off + i : -1;
}
// path id q = slot * B + b of a one-warp-per-path kernel inside the window (-1: none)
__device__ __forceinline__ int sub_path(const LtplDims& dm, int warps_per_cta) {
    const int i = blockIdx.x * warps_per_cta + (threadIdx.x >> 5);
    if (i >= LTPL_NSLOT * dm.sub_cnt) return -1;
    return (i / dm.sub_cnt) * dm.batch + dm.sub_off + i % dm.sub_cnt;
}

// ---------------------------------------------------------------------------------------------------------------------
// float64 helpers with NumPy operation order
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double sq_rn(double a) { return __dmul_rn(a, a); }

// np.power(ax - bx, 2) + np.power(ay - by, 2)
__device__ __forceinline__ double dist2_rn(double ax, double ay, double bx, double by) {
    return __dadd_rn(sq_rn(__dsub_rn(ax, bx)), sq_rn(__dsub_rn(ay, by)));
}

// 1 / sqrt(q) and 1 / x for VALUES (never for decisions): fp32 seed + two Newton steps in float64 (~2e-16 relative)
// instead of the emulated float64 rsqrt / division (~30-40 instructions each).  q, x > 0 and inside the fp32 range.
__device__ __forceinline__ double fast_rsqrt(double q) {
    double r = (double)rsqrtf((float)q);
    r = r * (1.5 - 0.5 * q * r * r);
    return r * (1.5 - 0.5 * q * r * r);
}
__device__ __forceinline__ double fast_rcp(double x) {
    double r = (double)__frcp_rn((float)x);
    r = r * (2.0 - x * r);
    return r * (2.0 - x * r);
}

// get_s_coord.py:102-121
__device__ __forceinline__ double angle3pt(double ax, double ay, double bx, double by, double cx, double cy) {
    double ang = atan2(cy - by, cx - bx) - atan2(ay - by, ax - bx);
    if (ang > LTPL_PI)
        ang -= 2 * LTPL_PI;
    else if (ang <= -LTPL_PI)
        ang += 2 * LTPL_PI;
    return ang;
}

// |angle3pt(pn, P, p1)| against |angle3pt(pn, P, p2)| (get_s_coord.py:60-77: which neighbour segment holds P).  The
// unsigned angle at P between (pn - P) and (p_i - P) is strictly decreasing in its cosine, so the comparison is decided
// on the two cosines whenever they differ by more than 1e-9 (orders of magnitude above the rounding of either
// formulation); only near-ties evaluate the reference's atan2 expression.  gt: ang1 > ang2, ge: ang1 >= ang2.
struct AngCmp {
    bool gt, ge;
};
// the reference's own expression (four atan2): only reached on near-ties, kept out of line (instruction cache)
__device__ __noinline__ AngCmp angle_cmp_exact(double2 pn, double px, double py, double2 p1, double2 p2) {
    const double a1 = fabs(angle3pt(pn.x, pn.y, px, py, p1.x, p1.y));
    const double a2 = fabs(angle3pt(pn.x, pn.y, px, py, p2.x, p2.y));
    AngCmp r;
    r.gt = a1 > a2;
    r.ge = a1 >= a2;
    return r;
}
__device__ __forceinline__ AngCmp angle_cmp(double2 pn, double px, double py, double2 p1, double2 p2) {
    const double ux = pn.x - px, uy = pn.y - py;
    const double v1x = p1.x - px, v1y = p1.y - py, v2x = p2.x - px, v2y = p2.y - py;
    const double un = ux * ux + uy * uy, n1 = v1x * v1x + v1y * v1y, n2 = v2x * v2x + v2y * v2y;
    AngCmp r;
    if (un > 0.0 && n1 > 0.0 && n2 > 0.0) {
        // (the cosines only have to be good to ~1e-12: the margin below is 1e-9)
        const double c1 = (ux * v1x + uy * v1y) * fast_rsqrt(n1), c2 = (ux * v2x + uy * v2y) * fast_rsqrt(n2);
        const double d = c1 - c2;
        if (d * d > 1e-18 * un) {
            r.gt = r.ge = (c1 < c2);
            return r;
        }
    }
    return angle_cmp_exact(pn, px, py, p1, p2);
}

// tph.normalize_psi
__device__ __forceinline__ double normalize_psi(double psi) {
    double a = fmod(fabs(psi), 2 * LTPL_PI);
    double out = (psi > 0.0) ? a : ((psi < 0.0) ? -a : 0.0);
    if (out >= LTPL_PI)
        out -= 2 * LTPL_PI;
    else if (out < -LTPL_PI)
        out += 2 * LTPL_PI;
    return out;
}

struct ArgMinD {
    double v;
    int i;
};

// first-minimum argmin over the warp (ties -> lower index), every lane gets the result
// v >= 0 (squared distances): the bit pattern of a non-negative double orders like the value, so the minimum is three
// 32-bit warp reductions (REDUX): high word, low word among the high-word winners, index among the value winners.
__device__ __forceinline__ ArgMinD warp_argmin(double v, int i) {
    const unsigned long long u = (unsigned long long)__double_as_longlong(v);
    const unsigned hi = (unsigned)(u >> 32), lo = (unsigned)u;
    const unsigned mh = __reduce_min_sync(LTPL_FULL, hi);
    const unsigned ml = __reduce_min_sync(LTPL_FULL, (hi == mh) ? lo : 0xffffffffu);
    const unsigned mi = __reduce_min_sync(LTPL_FULL, (hi == mh && lo == ml) ? (unsigned)i : 0xffffffffu);
    ArgMinD r;
    r.v = __longlong_as_double((long long)(((unsigned long long)mh << 32) | ml));
    r.i = (int)mi;
    return r;
}

// np.argmin of squared distances between pos and n points (closest_path_index.py:24-30, GIE:41-42, GB:341-345)
__device__ __noinline__ ArgMinD warp_closest_point(const double2* __restrict__ pts, int n, double px, double py,
                                                      int lane) {
    double bv = LTPL_INF;
    int bi = 0x7fffffff;
    #pragma unroll 1
    for (int i0 = lane; i0 < n; i0 += 128) {  // four loads in flight per lane; candidates still visited in index order
        double2 p[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) p[u] = pts[min(i0 + 32 * u, n - 1)];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int i = i0 + 32 * u;
            const double d = dist2_rn(p[u].x, p[u].y, px, py);
            if (i < n && d < bv) {
                bv = d;
                bi = i;
            }
        }
    }
    return warp_argmin(bv, bi);
}

// the same argmin for one of the lattice's own polylines: the grid cell of (px, py) bounds the nearest vertex (and every
// vertex tied with it) to <= 32 consecutive indices -> one distance per lane instead of a scan of the polyline; cells
// without a bound (far from the track) fall back to the scan.  Exact by construction (lattice_blob.nearest_grid).
__device__ __noinline__ ArgMinD warp_closest_point_grid(const LatDev& lt, const int* __restrict__ grid,
                                                           const double2* __restrict__ pts, int n, double px, double py,
                                                           int lane) {
    const double fx = floor((px - lt.grid_x0) * lt.grid_inv_cell), fy = floor((py - lt.grid_y0) * lt.grid_inv_cell);
    if (fx >= 0.0 && fy >= 0.0 && fx < (double)lt.grid_nx && fy < (double)lt.grid_ny) {
        const int ent = grid[(int)fy * lt.grid_nx + (int)fx];
        const int cnt = ent & 63;
        if (cnt) {
            int i = (ent >> 6) + lane;
            if (lt.grid_cyclic && i >= n) i -= n;
            double dv = LTPL_INF;
            if (lane < cnt) {
                const double2 p = pts[i];
                dv = dist2_rn(p.x, p.y, px, py);
            } else {
                i = 0x7fffffff;
            }
            return warp_argmin(dv, i);
        }
    }
    return warp_closest_point(pts, n, px, py, lane);
}

// ---- one query PER LANE -------------------------------------------------------------------------------------------
// The searches of a scenario (constant-segment ends, every object, every disc) are independent of each other; run one
// per lane, their dependent load -> compare -> load chains overlap instead of following each other warp-wide.
// Nearest vertex of this lane's position (active lanes): the candidates of its grid cell, serially; lanes whose cell has
// no bound are served one after the other by the warp-wide scan.
__device__ __forceinline__ int lanes_closest_point(const LatDev& lt, const int* __restrict__ grid,
                                                   const double2* __restrict__ pts, int n, double px, double py,
                                                   bool active, int lane) {
    int res = 0;
    bool fb = false;
    if (active) {
        const double fx = floor((px - lt.grid_x0) * lt.grid_inv_cell), fy = floor((py - lt.grid_y0) * lt.grid_inv_cell);
        int cnt = 0, first = 0;
        if (fx >= 0.0 && fy >= 0.0 && fx < (double)lt.grid_nx && fy < (double)lt.grid_ny) {
            const int ent = grid[(int)fy * lt.grid_nx + (int)fx];
            cnt = ent & 63;
            first = ent >> 6;
        }
        fb = (cnt == 0);
        double bv = LTPL_INF;
        int bi = 0x7fffffff;
        #pragma unroll 1
        for (int c = 0; c < cnt; ++c) {
            int i = first + c;
            if (lt.grid_cyclic && i >= n) i -= n;
            const double2 p = pts[i];
            const double dv = dist2_rn(p.x, p.y, px, py);
            if (dv < bv || (dv == bv && i < bi)) {   // first minimum in INDEX order (the candidates may wrap)
                bv = dv;
                bi = i;
            }
        }
        res = bi;
    }
    unsigned m = __ballot_sync(LTPL_FULL, fb);
    while (m) {
        const int src = __ffs(m) - 1;
        m &= m - 1;
        const double qx = __shfl_sync(LTPL_FULL, px, src), qy = __shfl_sync(LTPL_FULL, py, src);
        const ArgMinD r = warp_closest_point(pts, n, qx, qy, lane);
        if (lane == src) res = r.i;
    }
    return res;
}

// get_s_coord.py:8-99 behind the nearest vertex nb, on a CLOSED polyline with explicit s_array (s_array[0] <= 0.05, i.e.
// no leading-zero insertion): neighbour choice by the larger angle (:48-58), foot of the perpendicular, s; per lane
__device__ __forceinline__ double s_coord_from_vertex(const double2* __restrict__ pts, const double* __restrict__ s_arr,
                                                      int n, int nb, double px, double py) {
    int idx2 = nb + 1;
    if (idx2 > n - 1) idx2 = 0;
    const int a1 = (nb - 1 < 0) ? nb - 1 + n : nb - 1;
    const double2 pn = pts[nb], p1 = pts[a1], p2 = pts[idx2];
    double2 a, b;
    double sbase;
    if (angle_cmp(pn, px, py, p1, p2).gt) {
        a = p1;
        b = pn;
        sbase = s_arr[a1];
    } else {
        a = pn;
        b = p2;
        sbase = s_arr[nb];
    }
    const double bax = b.x - a.x, bay = b.y - a.y;
    const double t = __ddiv_rn(__dadd_rn(__dmul_rn(px - a.x, bax), __dmul_rn(py - a.y, bay)), __dadd_rn(sq_rn(bax), sq_rn(bay)));
    const double sx = __dadd_rn(a.x, __dmul_rn(t, bax));
    const double sy = __dadd_rn(a.y, __dmul_rn(t, bay));
    return __dadd_rn(sbase, sqrt(__dadd_rn(sq_rn(a.x - sx), sq_rn(a.y - sy))));
}

// check_inside_bounds.py:26-59 (warp-collective)
__device__ __noinline__ bool inside_bounds(const LatDev& lt, double px, double py, int lane) {
    int i0, i1;
    {
        // get_s_coord(centerline, pos, only_index=True, closed=True)[1]
        ArgMinD m = warp_closest_point_grid(lt, lt.grid_center, lt.center, lt.L, px, py, lane);
        int nb = m.i, n = lt.L;
        int idx1 = nb - 1, idx2 = nb + 1;
        if (idx2 > n - 1) idx2 = 0;
        int a1 = (idx1 < 0) ? idx1 + n : idx1;
        double2 pn = lt.center[nb], p1 = lt.center[a1], p2 = lt.center[idx2];
        if (angle_cmp(pn, px, py, p1, p2).ge) {
            i0 = a1;
            i1 = nb;
        } else {
            i0 = nb;
            i1 = idx2;
        }
    }
    // np.linspace(a, b) with 50 points: y[k] = k * ((b - a) / 49) + a, y[49] = b
    double2 c0 = lt.center[i0], c1 = lt.center[i1];
    double stx = __ddiv_rn(c1.x - c0.x, 49.0), sty = __ddiv_rn(c1.y - c0.y, 49.0);
    double bv = LTPL_INF;
    int bi = 0x7fffffff;
    #pragma unroll 1
    for (int k = lane; k < 50; k += 32) {
        double cx = (k == 49) ? c1.x : __dadd_rn(__dmul_rn((double)k, stx), c0.x);
        double cy = (k == 49) ? c1.y : __dadd_rn(__dmul_rn((double)k, sty), c0.y);
        double d = dist2_rn(cx, cy, px, py);
        if (d < bv) {
            bv = d;
            bi = k;
        }
    }
    ArgMinD m = warp_argmin(bv, bi);
    int k = m.i;
    double2 u0 = lt.bound1[i0], u1 = lt.bound1[i1], w0 = lt.bound2[i0], w1 = lt.bound2[i1];
    double b1x = (k == 49) ? u1.x : __dadd_rn(__dmul_rn((double)k, __ddiv_rn(u1.x - u0.x, 49.0)), u0.x);
    double b1y = (k == 49) ? u1.y : __dadd_rn(__dmul_rn((double)k, __ddiv_rn(u1.y - u0.y, 49.0)), u0.y);
    double b2x = (k == 49) ? w1.x : __dadd_rn(__dmul_rn((double)k, __ddiv_rn(w1.x - w0.x, 49.0)), w0.x);
    double b2y = (k == 49) ? w1.y : __dadd_rn(__dmul_rn((double)k, __ddiv_rn(w1.y - w0.y, 49.0)), w0.y);
    double d_track_2 = dist2_rn(b1x, b1y, b2x, b2y);
    double d_b1_2 = dist2_rn(b1x, b1y, px, py);
    double d_b2_2 = dist2_rn(b2x, b2y, px, py);
    return !(d_b1_2 > d_track_2 || d_b2_2 > d_track_2);
}

// check_inside_bounds.py:26-59 behind the nearest centre-line vertex nb: per lane.  The argmin over the 50 linspace points
// between the two centre-line vertices is taken over the six points around the foot of the perpendicular: the squared
// distance is a convex quadratic in the point index, every other point is further by >= 2 (|c1 - c0| / 49)^2 (orders of
// magnitude above the rounding of either evaluation); degenerate (nearly coincident) vertices scan all 50.
__device__ __forceinline__ bool inside_bounds_from_vertex(const LatDev& lt, int nb, double px, double py) {
    const int n = lt.L;
    int idx2 = nb + 1;
    if (idx2 > n - 1) idx2 = 0;
    const int a1 = (nb - 1 < 0) ? nb - 1 + n : nb - 1;
    int i0, i1;
    {
        const double2 pn = lt.center[nb], p1 = lt.center[a1], p2 = lt.center[idx2];
        if (angle_cmp(pn, px, py, p1, p2).ge) {
            i0 = a1;
            i1 = nb;
        } else {
            i0 = nb;
            i1 = idx2;
        }
    }
    const double2 c0 = lt.center[i0], c1 = lt.center[i1];
    const double2 u0 = lt.bound1[i0], u1 = lt.bound1[i1], w0 = lt.bound2[i0], w1 = lt.bound2[i1];
    const double stx = __ddiv_rn(c1.x - c0.x, 49.0), sty = __ddiv_rn(c1.y - c0.y, 49.0);
    const double ex = c1.x - c0.x, ey = c1.y - c0.y;
    const double den = ex * ex + ey * ey;
    int lo = 0, hi = 49;
    if (den > 1e-6) {
        double kc = ((px - c0.x) * ex + (py - c0.y) * ey) * fast_rcp(den) * 49.0;
        kc = fmin(fmax(kc, 0.0), 49.0);
        const int kf = (int)kc;
        lo = max(kf - 2, 0);
        hi = min(kf + 3, 49);
    }
    double bv = LTPL_INF;
    int k = 0;
    #pragma unroll 1
    for (int j = lo; j <= hi; ++j) {
        const double cx = (j == 49) ? c1.x : __dadd_rn(__dmul_rn((double)j, stx), c0.x);
        const double cy = (j == 49) ? c1.y : __dadd_rn(__dmul_rn((double)j, sty), c0.y);
        const double dv = dist2_rn(cx, cy, px, py);
        if (dv < bv) {   // first minimum
            bv = dv;
            k = j;
        }
    }
    const double b1x = (k == 49) ? u1.x : __dadd_rn(__dmul_rn((double)k, __ddiv_rn(u1.x - u0.x, 49.0)), u0.x);
    const double b1y = (k == 49) ? u1.y : __dadd_rn(__dmul_rn((double)k, __ddiv_rn(u1.y - u0.y, 49.0)), u0.y);
    const double b2x = (k == 49) ? w1.x : __dadd_rn(__dmul_rn((double)k, __ddiv_rn(w1.x - w0.x, 49.0)), w0.x);
    const double b2y = (k == 49) ? w1.y : __dadd_rn(__dmul_rn((double)k, __ddiv_rn(w1.y - w0.y, 49.0)), w0.y);
    const double d_track_2 = dist2_rn(b1x, b1y, b2x, b2y);
    const double d_b1_2 = dist2_rn(b1x, b1y, px, py);
    const double d_b2_2 = dist2_rn(b2x, b2y, px, py);
    return !(d_b1_2 > d_track_2 || d_b2_2 > d_track_2);
}

// planning-range membership of a layer (GB:704-709)
__device__ __forceinline__ bool layer_in_range(int x, int start, int end) {
    return (start < end) ? (x >= start && x <= end) : (x >= start || x <= end);
}

// np.interp(v, xp, fp) for increasing xp (clamped at both ends)
__device__ __forceinline__ double interp_table(double v, const double* __restrict__ xp, const double* __restrict__ fp,
                                               int n) {
    if (v <= xp[0]) return fp[0];
    if (v >= xp[n - 1]) return fp[n - 1];
    int j = 0;
    while (j < n - 2 && v >= xp[j + 1]) ++j;
    double slope = (fp[j + 1] - fp[j]) / (xp[j + 1] - xp[j]);
    return slope * (v - xp[j]) + fp[j];
}
