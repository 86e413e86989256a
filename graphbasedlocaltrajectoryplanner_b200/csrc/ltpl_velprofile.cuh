// ltpl_velprofile.cuh -- stand-alone velocity planner over [n_paths][n_points] arrays (ltpl_vel_plan_batch,
// ltpl_velprofile_batch = BASELINE.json config 5):
//   k_velprofile  tph.calc_vel_profile(closed=False, loc_gg mode), oracle/tph_port.py:463-538 (VPFB:194-227)
//   k_velbrake    tph.calc_vel_profile_brake, oracle/tph_port.py:659-732 (VPFB:229-255)
//   k_brakeprefix VpForwardBackward.check_brake_prefix (VPFB:86-139, ltpl_brake_prefix_batch): k_velbrake's chain with
//                 the old gg scale per path, cut where the speed reaches vel_max
//
// Throughput regime (100 k paths x 500 points): one LANE per path, one warp = 32 paths, the path arrays stream through
// shared memory in tiles of VD_H points x 32 paths (cp.async, transposing on the fly so that a lane reads its path down a
// conflict-free column).  Every point of k_velprofile takes the fp32 sweep steps of k_vel_res (VRSweep::fwd / bwd with the
// machine-table segment cache VRSeg, ltpl_vel_res.cuh); every point of k_velbrake the float64 brake_step of k_backup and
// k_emergency (ltpl_vel.cuh).  These kernels only add the tiling.
//   sweep 1 (forward):  kappa, el tiles in -> w tile -> fp32 scratch inside the caller's `ax` rows (4 bytes per point)
//   sweep 2 (backward): kappa, el, w tiles in -> final w; vx = sqrt(w) and ax = (w1 - w0) / (2 el) leave through the tiles
// HBM traffic per point: 2 x 16 B in (kappa, el: twice) + 4 B out + 4 B in (w) + 16 B out (vx, ax) = 56 B
// (algorithmic minimum 32 B: the w profile of 100 k x 500 points does not fit on the chip between the sweeps).
// Per-point friction (GG) adds 2 x 16 B in (ax_max, ay_max in both sweeps; algorithmic + 16 B).
#pragma once
#include "ltpl_vel_res.cuh"

#define VD_W 33
#ifndef VD_H
#define VD_H 32                            // points per tile (power of two <= 32)
#endif
#define VD_TILE (VD_H * VD_W)
#define VD_SMEM_BYTES (2 * VD_TILE * 8 + VD_TILE * 4)   // kappa, el (float64; reused for vx, ax), w (fp32)

// General layout of ltpl_vel_plan_batch: the kernels take it as a third parameter behind the parent's two, so the dense
// constant-friction instances of k_velprofile read their parameters where they always did.
struct VdLayout {
    const int32_t* n_pts;   // [n_paths] points per path; NULL: n_points each
    const double* gg;       // [n_paths][n_points][2] ax_max, ay_max; NULL: params.gg_ax / gg_ay
    int64_t k_s, e_s, g_s, o_s;   // row strides in elements: kappa, el, gg, vx / ax
};

// general layout: dynamic shared memory behind the tiles of VD_SMEM_BYTES
//   GG: ax_max, ay_max tiles (float64);  then s_n[32] (points of each path of the warp, 0: none to read) and
//   s_o[32] (output points of each row: n_points inside the batch, 0 behind it)
__host__ __device__ constexpr int vd_smem_general(bool gg) { return VD_SMEM_BYTES + (gg ? 2 * VD_TILE * 8 : 0) + 64 * 4; }
// k_velbrake: kappa, el (reused for ax, vx), GG tiles, s_n, s_o
__host__ __device__ constexpr int vd_smem_brake(bool gg) { return 2 * VD_TILE * 8 + (gg ? 2 * VD_TILE * 8 : 0) + 64 * 4; }

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

// General layout: row r of the warp (path path0 + r) starts at base + rs (path0 + r); its point p is the element step p
// of the row (step 2: one column of the gg pairs).  Only points p < lim[r] - cut are read (lim: s_n; cut 1 for el,
// whose last element is never used).  MIR: the tile's point p holds the row's mirror point lim[r] - 1 - p -- the
// per-point friction the backward sweep reads (tph does not flip it, vr_backward).
template <bool MIR = false, typename T>
__device__ __forceinline__ void vd_load_rows(T* tile, const T* base, int64_t rs, int step, const int* lim, int cut,
                                             int path0, int p0, int lane) {
    const int pt = lane % VD_H, sub = lane / VD_H;
    const int p = p0 + pt;
#pragma unroll 4
    for (int r = sub; r < 32; r += 32 / VD_H) {
        const int m = lim[r];
        if (p < m - cut) {
            const T* src = base + (size_t)(path0 + r) * rs + (size_t)step * (MIR ? m - 1 - p : p);
            if constexpr (sizeof(T) == 8)
                vd_cp_async8(&tile[pt * VD_W + r], src);
            else
                vd_cp_async4(&tile[pt * VD_W + r], src);
        }
    }
}
// general layout: points p < lim[r] of row r
template <typename T>
__device__ __forceinline__ void vd_store_rows(const T* tile, T* base, int64_t rs, const int* lim, int path0, int p0,
                                              int lane) {
    const int pt = lane % VD_H, sub = lane / VD_H;
    const int p = p0 + pt;
#pragma unroll 4
    for (int r = sub; r < 32; r += 32 / VD_H) {
        if (p < lim[r]) base[(size_t)(path0 + r) * rs + p] = tile[pt * VD_W + r];
    }
}

// General layout: the lane's points n_i (0 behind the batch and for a length out of [2, n_points]: `bad` then) into
// s_n, the output points of its row into s_o.  Returns n_i.
template <bool RAGGED>
__device__ __forceinline__ int vd_lengths(const LtplVelBatch& vb, const VdLayout& va, int path0, int lane, int* s_n,
                                          int* s_o, bool& bad) {
    const int n = vb.n_points;
    const bool in = path0 + lane < vb.n_paths;
    int m = in ? n : 0;
    if constexpr (RAGGED) {
        if (in && va.n_pts) m = va.n_pts[path0 + lane];
    }
    bad = in && (m < 2 || m > n);
    const int n_i = bad ? 0 : m;
    s_n[lane] = n_i;
    s_o[lane] = in ? n : 0;
    return n_i;
}

// EXP1: friction-ellipse exponent 1.0 (no pow on the chain).  GG: per-point friction va.gg (times gg_scale), else the
// constant params.gg_ax / gg_ay (times gg_scale).  RAGGED: a length per path (va.n_pts) or row strides other than
// n_points.  <EXP1, false, false> is the dense solver: rows of n_points, the parameter vb only.
// RAGGED: the forward sweep is aligned at p = 0, a lane stops storing behind its end and clamps v_end at its own last
// point; the backward sweep walks from n_points - 1 down and a lane starts at its last point.  Outputs behind a path's
// end are 0; a path whose length is out of range gets a row of NaN.
template <bool EXP1, bool GG, bool RAGGED>
__global__ void __launch_bounds__(32)
k_velprofile(const __grid_constant__ LtplParams prm, const __grid_constant__ LtplVelBatch vb,
             const __grid_constant__ VdLayout va) {
    constexpr bool GEN = GG || RAGGED;   // general layout
    extern __shared__ __align__(16) unsigned char vd_smem[];
    double* t_k = reinterpret_cast<double*>(vd_smem);
    double* t_e = t_k + VD_TILE;
    float* t_w = reinterpret_cast<float*>(t_e + VD_TILE);
    double* t_v = t_e;   // vx replaces el in place (the element's el is consumed before vx is written)
    double* t_a = t_k;   // ax replaces kappa in place
    double* t_gx = reinterpret_cast<double*>(t_w + VD_TILE);   // GG: ax_max, ay_max of the tile's points
    double* t_gy = t_gx + VD_TILE;
    int* s_n = reinterpret_cast<int*>(GG ? t_gy + VD_TILE : t_gx);   // GEN
    int* s_o = s_n + 32;
    __shared__ float s_tab[4 * VR_TAB];
    int n_lane = 0;      // GEN: this lane's points
    bool bad = false;    // GEN: its length is out of range
    if constexpr (GEN) n_lane = vd_lengths<RAGGED>(vb, va, blockIdx.x * 32, threadIdx.x, s_n, s_o, bad);
    vr_stage_axm(prm, s_tab);
    __syncthreads();
    const int lane = threadIdx.x;
    const int path0 = blockIdx.x * 32;
    const int n = vb.n_points;
    const int n_i = GEN ? n_lane : n;   // this lane's points
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
    int n_warp = n;   // RAGGED: the forward sweep ends with the warp's longest path
    if constexpr (RAGGED) n_warp = (int)__reduce_max_sync(LTPL_FULL, (unsigned)n_i);

    // ---- forward sweep (tph.__solver_fb_acc_profile(backwards=False)) ----
    VRSweep f;   // starts at p = 0
    VRSeg seg;
    seg.load(c, 1);
    float e_prev = 0.0f;
    for (int tl = 0; tl < ntile; ++tl) {
        const int p0 = tl * VD_H;
        if constexpr (RAGGED) {
            if (p0 >= n_warp) break;
        }
        if constexpr (GEN) {
            vd_load_rows(t_k, vb.kappa, va.k_s, 1, s_n, 0, path0, p0, lane);
            vd_load_rows(t_e, vb.el, va.e_s, 1, s_n, 1, path0, p0, lane);
            if constexpr (GG) {
                vd_load_rows(t_gx, va.gg, va.g_s, 2, s_n, 0, path0, p0, lane);
                vd_load_rows(t_gy, va.gg + 1, va.g_s, 2, s_n, 0, path0, p0, lane);
            }
        } else {
            vd_load(t_k, vb.kappa, path0, vb.n_paths, n, p0, lane);
            vd_load(t_e, vb.el, path0, vb.n_paths, n, p0, lane);
        }
        vd_cp_async_wait_all();
        __syncwarp();
#pragma unroll 2
        for (int k = 0; k < VD_H; ++k) {
            const int p = p0 + k;
            const bool in = p < n_i;   // warp uniform unless RAGGED
            // GG: the point's own friction (tph: p_ggv[i] of the unflipped arrays)
            const double iay = GG ? 1.0 / (t_gy[k * VD_W + lane] * prm.gg_scale) : inv_ay;
            const float axq = GG ? (float)(t_gx[k * VD_W + lane] * prm.gg_scale) : c.ax_max;
            const float kq = (float)(fabs(t_k[k * VD_W + lane]) * iay);
            const float e2 = (float)(2.0 * t_e[k * VD_W + lane]);
            float w;
            if (p == 0) {
                w = vr_w_start(kq, wmax, wcap);
                f.start(w, kq, axq);
            } else {
                // points behind the path end step on without storing; nothing reads their state
                w = f.fwd<EXP1>(c, seg, kq, axq, e_prev, wmax, live && in);
            }
            e_prev = e2;
            if (p == n_i - 1) vr_clamp_end(w, we);
            if (in) t_w[k * VD_W + lane] = w;
        }
        __syncwarp();
        if constexpr (GEN)
            vd_store_rows(t_w, wscr, 2 * va.o_s, s_n, path0, p0, lane);
        else
            vd_store_w(t_w, wscr, path0, vb.n_paths, n, p0, lane);
        __syncwarp();
    }

    // ---- backward sweep (flipped arrays, mode 'decel_backw', one look-ahead correction); vx, ax on the way ----
    VRSweep b;   // starts at p = n_i - 1
    float w_next = 0.0f;
    for (int tl = ntile - 1; tl >= 0; --tl) {
        const int p0 = tl * VD_H;
        if constexpr (GEN) {
            vd_load_rows(t_k, vb.kappa, va.k_s, 1, s_n, 0, path0, p0, lane);
            vd_load_rows(t_e, vb.el, va.e_s, 1, s_n, 1, path0, p0, lane);
            vd_load_rows(t_w, wscr, 2 * va.o_s, 1, s_n, 0, path0, p0, lane);
            if constexpr (GG) {
                vd_load_rows<true>(t_gx, va.gg, va.g_s, 2, s_n, 0, path0, p0, lane);
                vd_load_rows<true>(t_gy, va.gg + 1, va.g_s, 2, s_n, 0, path0, p0, lane);
            }
        } else {
            vd_load(t_k, vb.kappa, path0, vb.n_paths, n, p0, lane);
            vd_load(t_e, vb.el, path0, vb.n_paths, n, p0, lane);
            vd_load_w(t_w, wscr, path0, vb.n_paths, n, p0, lane);
        }
        vd_cp_async_wait_all();
        __syncwarp();
#pragma unroll 2
        for (int k = VD_H - 1; k >= 0; --k) {
            const int p = p0 + k;
            if (p < n) {   // warp uniform
                // GG: the friction of the mirror point n_i - 1 - p (vr_backward)
                const double iay = GG ? 1.0 / (t_gy[k * VD_W + lane] * prm.gg_scale) : inv_ay;
                const float axq = GG ? (float)(t_gx[k * VD_W + lane] * prm.gg_scale) : c.ax_max;
                const float kq = (float)(fabs(t_k[k * VD_W + lane]) * iay);
                const float e2 = (float)(2.0 * t_e[k * VD_W + lane]);
                const float o_n = t_w[k * VD_W + lane];
                float wv = o_n, a_out = 0.0f;
                if (p < n_i - 1) {
                    wv = b.bwd<EXP1>(c, o_n, kq, axq, e2, wmax);
                    a_out = (w_next - wv) * vr_rcp(e2);
                } else {
                    b.start(o_n, kq, axq);   // (RAGGED: again at every point behind the end, last at n_i - 1)
                }
                if constexpr (GEN) {   // 0 behind the path's end, NaN for a length out of range
                    const double z = bad ? CUDART_NAN : 0.0;
                    t_v[k * VD_W + lane] = (p < n_i) ? (double)vr_sqrt(wv) : z;
                    t_a[k * VD_W + lane] = (p < n_i) ? (double)a_out : z;
                } else {
                    t_v[k * VD_W + lane] = (double)vr_sqrt(wv);
                    t_a[k * VD_W + lane] = (double)a_out;
                }
                w_next = wv;
            }
        }
        __syncwarp();
        if constexpr (GEN) {
            vd_store_rows(t_v, vb.vx, va.o_s, s_o, path0, p0, lane);
            vd_store_rows(t_a, vb.ax, va.o_s, s_o, path0, p0, lane);
        } else {
            vd_store(t_v, vb.vx, path0, vb.n_paths, n, p0, lane);
            vd_store(t_a, vb.ax, path0, vb.n_paths, n, p0, lane);
        }
        __syncwarp();
    }
}

// tph.calc_vel_profile_brake (VPFB:229-255: raw friction, no gg_scale): from max(v_start, 0) one float64 brake_step per
// point (the step of k_backup and k_emergency) until the radicand turns negative; from there on vx and ax are 0.
// ax = (w1 - w0) / (2 el), 0 at the last point.  Any length per path and row strides (general layout); GG: per-point
// friction va.gg, else params.gg_ax / gg_ay.
template <bool GG>
__global__ void __launch_bounds__(32)
k_velbrake(const __grid_constant__ LtplParams prm, const __grid_constant__ LtplVelBatch vb,
           const __grid_constant__ VdLayout va) {
    extern __shared__ __align__(16) unsigned char vd_smem[];
    double* t_k = reinterpret_cast<double*>(vd_smem);
    double* t_e = t_k + VD_TILE;
    double* t_v = t_e;   // vx replaces el in place
    double* t_a = t_k;   // ax replaces kappa in place
    double* t_gx = t_e + VD_TILE;
    double* t_gy = t_gx + VD_TILE;
    int* s_n = reinterpret_cast<int*>(GG ? t_gy + VD_TILE : t_gx);
    int* s_o = s_n + 32;
    const int lane = threadIdx.x;
    const int path0 = blockIdx.x * 32;
    const int n = vb.n_points;
    bool bad;
    const int n_i = vd_lengths<true>(vb, va, path0, lane, s_n, s_o, bad);
    __syncwarp();
    const double dmq = prm.drag_coeff / prm.m_veh, inv_ay = 1.0 / prm.gg_ay;
    const double v0 = (path0 + lane < vb.n_paths) ? fmax(vb.v_start[path0 + lane], 0.0) : 0.0;
    double w = v0 * v0;
    bool stopped = false;
    const int ntile = (n + VD_H - 1) / VD_H;
    for (int tl = 0; tl < ntile; ++tl) {
        const int p0 = tl * VD_H;
        // the inputs of a tile are read while some lane of the warp still brakes inside it
        if (!__all_sync(LTPL_FULL, stopped || p0 >= n_i - 1)) {
            vd_load_rows(t_k, vb.kappa, va.k_s, 1, s_n, 0, path0, p0, lane);
            vd_load_rows(t_e, vb.el, va.e_s, 1, s_n, 1, path0, p0, lane);
            if constexpr (GG) {
                vd_load_rows(t_gx, va.gg, va.g_s, 2, s_n, 0, path0, p0, lane);
                vd_load_rows(t_gy, va.gg + 1, va.g_s, 2, s_n, 0, path0, p0, lane);
            }
            vd_cp_async_wait_all();
        }
        __syncwarp();
#pragma unroll 1
        for (int k = 0; k < VD_H; ++k) {
            const int p = p0 + k;
            double v = 0.0, a = 0.0;
            if (p < n_i) {
                v = (p == 0) ? v0 : sqrt(w);
                if (p < n_i - 1 && !stopped) {
                    const double kabs = fabs(t_k[k * VD_W + lane]), ds = t_e[k * VD_W + lane];
                    const double nx = GG ? brake_step(w, kabs, t_gx[k * VD_W + lane], 1.0 / t_gy[k * VD_W + lane],
                                                      prm.dyn_model_exp, dmq, ds)
                                         : brake_step(w, kabs, prm.gg_ax, inv_ay, prm.dyn_model_exp, dmq, ds);
                    double wn = 0.0;
                    if (nx < 0.0)   // negative radicand: standstill, the rest of the profile stays 0
                        stopped = true;
                    else
                        wn = nx;
                    a = (wn - w) / (2 * ds);
                    w = wn;
                }
            }
            if (bad) v = a = CUDART_NAN;
            t_v[k * VD_W + lane] = v;
            t_a[k * VD_W + lane] = a;
        }
        __syncwarp();
        vd_store_rows(t_v, vb.vx, va.o_s, s_o, path0, p0, lane);
        vd_store_rows(t_a, vb.ax, va.o_s, s_o, path0, p0, lane);
        __syncwarp();
    }
}

// k_brakeprefix: k_velbrake's shared memory (kappa, el reused for the prefix values, GG tiles, s_n, s_o), then s_c[32]
// (course points of each row: where its brake part starts) and s_w[32] (prefix positions from there to the row's end)
__host__ __device__ constexpr int vd_smem_prefix(bool gg) { return vd_smem_brake(gg) + 64 * 4; }

// points p < lim[r] of row r at base + rs (path0 + r) + off[r] + p: vd_store_rows with a start offset per row
__device__ __forceinline__ void bp_store_rows(const double* tile, double* base, int64_t rs, const int* off,
                                              const int* lim, int path0, int p0, int lane) {
    const int pt = lane % VD_H, sub = lane / VD_H;
    const int p = p0 + pt;
#pragma unroll 4
    for (int r = sub; r < 32; r += 32 / VD_H) {
        if (p < lim[r]) base[(size_t)(path0 + r) * rs + off[r] + p] = tile[pt * VD_W + r];
    }
}

// VpForwardBackward.check_brake_prefix (VPFB:86-139) with the instance's old_gg_scale per path (LtplBrakePrefix).
// A lane whose vel_plan exceeds vel_max + 0.1 runs k_velbrake's float64 chain (brake_step, friction times its old scale:
// gx old and 1 / (gy old), as tph reads loc_gg * old_gg_scale) and stops at its cut: the first point at or below vel_max
// (np.argmax; none, or point 0: n - 1).  Row layout: vel_course[:c] (first pass, through the kappa tile), the brake
// points [0, idx) from position c on, zeros up to C + n_points - 1.  Tile loads stop once every lane has cut.
template <bool GG>
__global__ void __launch_bounds__(32)
k_brakeprefix(const __grid_constant__ LtplParams prm, const __grid_constant__ LtplBrakePrefix bp) {
    extern __shared__ __align__(16) unsigned char vd_smem[];
    double* t_k = reinterpret_cast<double*>(vd_smem);
    double* t_e = t_k + VD_TILE;
    double* t_v = t_e;   // the prefix values replace el in place
    double* t_c = t_k;   // the course passes through the kappa tile before the brake pass
    double* t_gx = t_e + VD_TILE;
    double* t_gy = t_gx + VD_TILE;
    int* s_n = reinterpret_cast<int*>(GG ? t_gy + VD_TILE : t_gx);
    int* s_o = s_n + 32;
    int* s_c = s_o + 32;
    int* s_w = s_c + 32;
    const int lane = threadIdx.x;
    const int path0 = blockIdx.x * 32;
    const int i = path0 + lane;
    const bool in = i < bp.n_paths;
    LtplVelBatch vb = {};
    vb.n_paths = bp.n_paths;
    vb.n_points = bp.n_points;
    VdLayout va = {};
    va.n_pts = bp.n_pts;
    bool bad;
    const int n_i = vd_lengths<true>(vb, va, path0, lane, s_n, s_o, bad);
    const int C = bp.n_course_cap;
    const int W = C + bp.n_points - 1;   // prefix positions per row
    int c_i = in ? C : 0;
    if (in && bp.n_course) c_i = bp.n_course[i];
    if (in && (c_i < 0 || c_i > C)) bad = true;
    if (bad) c_i = 0;
    s_c[lane] = c_i;
    s_w[lane] = in ? W - c_i : 0;
    const double vel_max = prm.vel_max;
    const double vp = in ? bp.vel_plan[i] : 0.0;
    const double old = in ? bp.old_gg_scale[i] : 1.0;
    const bool brake = in && !bad && vp > vel_max + 0.1;
    __syncwarp();

    // ---- vel_course[:c] ----
    for (int p0 = 0; p0 < C; p0 += VD_H) {
        vd_load_rows(t_c, bp.vel_course, bp.vel_course_s, 1, s_c, 0, path0, p0, lane);
        vd_cp_async_wait_all();
        __syncwarp();
        vd_store_rows(t_c, bp.vx_prefix, bp.vx_prefix_s, s_c, path0, p0, lane);
        __syncwarp();
    }

    // ---- brake points [0, idx) from position c on, then zeros ----
    const double dmq = prm.drag_coeff / prm.m_veh;
    const double ax_c = prm.gg_ax * old, iay_c = 1.0 / (prm.gg_ay * old);
    const double v0 = fmax(vp, 0.0);
    double w = v0 * v0;
    bool stopped = false;
    bool done = !brake;    // the lane has cut (or does not brake)
    bool nocut = false;    // point 0 is at or below vel_max: np.argmax gives 0, idx = n - 1
    int idx = 0;
    double vs = vp;
    // the cut can fall on point n_points - 1, one behind the last prefix position when C = 0: the loop walks every point
    // as well as every position (bp_store_rows stores positions < W only)
    const int ntile = (max(W, bp.n_points) + VD_H - 1) / VD_H;
    for (int tl = 0; tl < ntile; ++tl) {
        const int p0 = tl * VD_H;
        // the inputs of a tile are read while some lane of the warp still brakes inside it
        if (!__all_sync(LTPL_FULL, done || p0 >= n_i - 1)) {
            vd_load_rows(t_k, bp.kappa, bp.kappa_s, 1, s_n, 0, path0, p0, lane);
            vd_load_rows(t_e, bp.el, bp.el_s, 1, s_n, 1, path0, p0, lane);
            if constexpr (GG) {
                vd_load_rows(t_gx, bp.gg, bp.gg_s, 2, s_n, 0, path0, p0, lane);
                vd_load_rows(t_gy, bp.gg + 1, bp.gg_s, 2, s_n, 0, path0, p0, lane);
            }
            vd_cp_async_wait_all();
        }
        __syncwarp();
#pragma unroll 1
        for (int k = 0; k < VD_H; ++k) {
            const int p = p0 + k;
            double v = 0.0;
            if (!done) {
                v = (p == 0) ? v0 : sqrt(w);
                if (v <= vel_max && !nocut) {
                    if (p == 0)
                        nocut = true;
                    else
                        done = true;
                }
                if (p == n_i - 1) done = true;
                if (done) {   // the cut: vx_decel[idx] starts the next profile and is not part of the prefix
                    idx = p;
                    vs = v;
                    v = 0.0;
                } else if (!stopped) {
                    const double kabs = fabs(t_k[k * VD_W + lane]), ds = t_e[k * VD_W + lane];
                    const double nx = GG ? brake_step(w, kabs, t_gx[k * VD_W + lane] * old,
                                                      1.0 / (t_gy[k * VD_W + lane] * old), prm.dyn_model_exp, dmq, ds)
                                         : brake_step(w, kabs, ax_c, iay_c, prm.dyn_model_exp, dmq, ds);
                    if (nx < 0.0)   // negative radicand: standstill, the rest of the profile stays 0
                        stopped = true;
                    w = nx < 0.0 ? 0.0 : nx;
                }
            }
            if (bad) v = CUDART_NAN;
            t_v[k * VD_W + lane] = v;
        }
        __syncwarp();
        bp_store_rows(t_v, bp.vx_prefix, bp.vx_prefix_s, s_c, s_w, path0, p0, lane);
        __syncwarp();
    }
    if (in) {
        if (bad) {   // the memory stays
            bp.n_prefix[i] = bp.pref_idx[i] = -1;
            bp.vel_start[i] = CUDART_NAN;
        } else {
            bp.n_prefix[i] = c_i + idx;
            bp.pref_idx[i] = idx;
            bp.vel_start[i] = vs;
            if (!brake) bp.old_gg_scale[i] = prm.gg_scale;
        }
    }
}
