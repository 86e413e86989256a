// ltpl_velprofile.cuh -- k_velprofile: stand-alone forward/backward ggv solver over dense [n_paths][n_points] arrays
// (BASELINE.json config 5; tph.calc_vel_profile(closed=False, loc_gg mode), oracle/tph_port.py:463-538).
//
// Throughput regime (100 k paths x 500 points): one LANE per path, one warp = 32 paths, the path arrays stream through
// shared memory in tiles of VD_H points x 32 paths (cp.async, transposing on the fly so that a lane reads its path down a
// conflict-free column).  The recurrences are the fp32 steps of ltpl_vel_res.cuh (w = v^2, branch-free, machine-table
// segment cached in registers with a warp-uniform miss path).
//   sweep 1 (forward):  kappa, el tiles in -> w tile -> fp32 scratch inside the caller's `ax` rows (4 bytes per point)
//   sweep 2 (backward): kappa, el, w tiles in -> final w; vx = sqrt(w) and ax = (w1 - w0) / (2 el) leave through the tiles
// HBM traffic per point: 2 x 16 B in (kappa, el: twice) + 4 B out + 4 B in (w) + 16 B out (vx, ax) = 56 B
// (algorithmic minimum 32 B: the w profile of 100 k x 500 points does not fit on the chip between the sweeps).
#pragma once
#include "ltpl_vel_res.cuh"

#define VD_W 33
#ifndef VD_H
#define VD_H 32                            // points per tile (power of two <= 32)
#endif
#define VD_TILE (VD_H * VD_W)
#define VD_SMEM_BYTES (2 * VD_TILE * 8 + VD_TILE * 4)   // kappa, el (float64; reused for vx, ax), w (fp32)

__device__ __forceinline__ void vd_cp_async8(void* smem_dst, const void* gsrc) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" ::"r"(d), "l"(gsrc));
}
__device__ __forceinline__ void vd_cp_async4(void* smem_dst, const void* gsrc) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(d), "l"(gsrc));
}
__device__ __forceinline__ void vd_cp_async_wait_all() {
    asm volatile("cp.async.commit_group;\n" ::);
    asm volatile("cp.async.wait_group 0;\n" ::);
}

// one request covers 32 / VD_H path rows x VD_H consecutive points
__device__ __forceinline__ void vd_load(double* tile, const double* base, int path0, int n_paths, int n_points, int p0,
                                        int lane) {
    const int pt = lane % VD_H, sub = lane / VD_H;
#pragma unroll 4
    for (int r = sub; r < 32; r += 32 / VD_H) {
        if (path0 + r < n_paths && p0 + pt < n_points)
            vd_cp_async8(&tile[pt * VD_W + r], base + (size_t)(path0 + r) * n_points + p0 + pt);
    }
}
__device__ __forceinline__ void vd_store(const double* tile, double* base, int path0, int n_paths, int n_points, int p0,
                                         int lane) {
    const int pt = lane % VD_H, sub = lane / VD_H;
#pragma unroll 4
    for (int r = sub; r < 32; r += 32 / VD_H) {
        if (path0 + r < n_paths && p0 + pt < n_points)
            base[(size_t)(path0 + r) * n_points + p0 + pt] = tile[pt * VD_W + r];
    }
}
// fp32 scratch rows: path i keeps w[p] at float index p of its `ax` row (row stride 2 n_points floats)
__device__ __forceinline__ void vd_load_w(float* tile, const float* base, int path0, int n_paths, int n_points, int p0,
                                          int lane) {
    const int pt = lane % VD_H, sub = lane / VD_H;
#pragma unroll 4
    for (int r = sub; r < 32; r += 32 / VD_H) {
        if (path0 + r < n_paths && p0 + pt < n_points)
            vd_cp_async4(&tile[pt * VD_W + r], base + (size_t)(path0 + r) * 2 * n_points + p0 + pt);
    }
}
__device__ __forceinline__ void vd_store_w(const float* tile, float* base, int path0, int n_paths, int n_points, int p0,
                                           int lane) {
    const int pt = lane % VD_H, sub = lane / VD_H;
#pragma unroll 4
    for (int r = sub; r < 32; r += 32 / VD_H) {
        if (path0 + r < n_paths && p0 + pt < n_points)
            base[(size_t)(path0 + r) * 2 * n_points + p0 + pt] = tile[pt * VD_W + r];
    }
}

template <bool EXP1>
__global__ void __launch_bounds__(32)
k_velprofile(const __grid_constant__ LtplParams prm, const __grid_constant__ LtplVelBatch vb) {
    extern __shared__ __align__(16) unsigned char vd_smem[];
    double* t_k = reinterpret_cast<double*>(vd_smem);
    double* t_e = t_k + VD_TILE;
    float* t_w = reinterpret_cast<float*>(t_e + VD_TILE);
    double* t_v = t_e;   // vx replaces el in place (the element's el is consumed before vx is written)
    double* t_a = t_k;   // ax replaces kappa in place
    __shared__ float s_tab[4 * VR_TAB];
    vr_stage_axm(prm, s_tab);
    __syncthreads();
    const int lane = threadIdx.x;
    const int path0 = blockIdx.x * 32;
    const int n = vb.n_points;
    const bool live = path0 + lane < vb.n_paths;
    const VRCfg c = vr_make_cfg(prm, s_tab);
    const float wmax = (float)(prm.vel_max * prm.vel_max);
    const double inv_ay = 1.0 / (prm.gg_ay * prm.gg_scale);
    double vs = live ? vb.v_start[path0 + lane] : 0.0;
    double ve = live ? vb.v_end[path0 + lane] : 0.0;
    if (vs < 0.0) vs = 0.0;
    if (ve < 0.0) ve = 0.0;
    const float wcap = (float)(vs * vs), we = (float)(ve * ve);
    float* wscr = reinterpret_cast<float*>(vb.ax);
    const int ntile = (n + VD_H - 1) / VD_H;

    // ---- forward sweep (tph.__solver_fb_acc_profile(backwards=False)) ----
    float cur = 0.0f, o_prev = 0.0f, k_prev = 0.0f, e_prev = 0.0f;
    bool prev_rise = false, active = false;
    int sg = 1;
    float xlo = c.xl[1], xhi = c.xl[2], x0 = c.x0[1], f0 = c.f0[1], sl = c.sl[1];
    for (int tl = 0; tl < ntile; ++tl) {
        const int p0 = tl * VD_H;
        vd_load(t_k, vb.kappa, path0, vb.n_paths, n, p0, lane);
        vd_load(t_e, vb.el, path0, vb.n_paths, n, p0, lane);
        vd_cp_async_wait_all();
        __syncwarp();
#pragma unroll 2
        for (int k = 0; k < VD_H; ++k) {
            const int p = p0 + k;
            const bool in = p < n;   // warp uniform
            const float kq = (float)(fabs(t_k[k * VD_W + lane]) * inv_ay);
            const float e2 = (float)(2.0 * t_e[k * VD_W + lane]);
            const float o_n = fminf(vr_rcp(kq), wmax);
            float nxt;
            if (p == 0) {
                nxt = fminf(o_n, wcap);
            } else {
                const bool rise = o_n > o_prev;
                active = active || (rise && !prev_rise);
                const float v = vr_sqrt(fmaxf(cur, 0.0f));
                const bool need = live && in && active;
                bool miss = need && !(v >= xlo && v < xhi);
                while (__any_sync(LTPL_FULL, miss)) {
                    if (miss) sg += (v >= xhi) ? 1 : -1;
                    xlo = c.xl[sg];
                    xhi = c.xl[sg + 1];
                    x0 = c.x0[sg];
                    f0 = c.f0[sg];
                    sl = c.sl[sg];
                    miss = need && !(v >= xlo && v < xhi);
                }
                const float a_t = vr_tire<EXP1>(c, cur, k_prev, c.ax_max);
                const float a = fmaf(-cur, c.dm, fminf(a_t, fmaf(sl, v - x0, f0)));
                const float wn = fmaf(a, e_prev, cur);
                nxt = active ? fminf(wn, o_n) : o_n;
                active = active && !(wn > wmax);
                prev_rise = rise;
            }
            if (in) {
                o_prev = (p == 0) ? nxt : o_n;
                cur = nxt;
                k_prev = kq;
                e_prev = e2;
                t_w[k * VD_W + lane] = (p == n - 1 && nxt > we) ? we : nxt;   // v[-1] = min(v[-1], v_end)
            }
        }
        __syncwarp();
        vd_store_w(t_w, wscr, path0, vb.n_paths, n, p0, lane);
        __syncwarp();
    }

    // ---- backward sweep (flipped arrays, mode 'decel_backw', one look-ahead correction); vx, ax on the way ----
    float k_p = 0.0f, w_next = 0.0f;
    prev_rise = false;
    active = false;
    for (int tl = ntile - 1; tl >= 0; --tl) {
        const int p0 = tl * VD_H;
        vd_load(t_k, vb.kappa, path0, vb.n_paths, n, p0, lane);
        vd_load(t_e, vb.el, path0, vb.n_paths, n, p0, lane);
        vd_load_w(t_w, wscr, path0, vb.n_paths, n, p0, lane);
        vd_cp_async_wait_all();
        __syncwarp();
#pragma unroll 2
        for (int k = VD_H - 1; k >= 0; --k) {
            const int p = p0 + k;
            if (p < n) {   // warp uniform
                const float kq = (float)(fabs(t_k[k * VD_W + lane]) * inv_ay);
                const float e2 = (float)(2.0 * t_e[k * VD_W + lane]);
                const float o_n = t_w[k * VD_W + lane];
                float wv = o_n, a_out = 0.0f;
                if (p < n - 1) {
                    const bool rise = o_n > o_prev;
                    active = active || (rise && !prev_rise);
                    const float a = fmaf(cur, c.dm, vr_tire<EXP1>(c, cur, k_p, c.ax_max));
                    float wn = fmaf(a, e2, cur);
                    const float a2 = fmaf(wn, c.dm, vr_tire<EXP1>(c, wn, kq, c.ax_max));
                    wn = fminf(wn, fmaf(a2, e2, cur));
                    wv = active ? fminf(wn, o_n) : o_n;
                    active = active && !(wn > wmax);
                    prev_rise = rise;
                    a_out = (w_next - wv) * vr_rcp(e2);
                }
                t_v[k * VD_W + lane] = (double)vr_sqrt(wv);
                t_a[k * VD_W + lane] = (double)a_out;
                cur = wv;
                o_prev = o_n;
                k_p = kq;
                w_next = wv;
            }
        }
        __syncwarp();
        vd_store(t_v, vb.vx, path0, vb.n_paths, n, p0, lane);
        vd_store(t_a, vb.ax, path0, vb.n_paths, n, p0, lane);
        __syncwarp();
    }
}
