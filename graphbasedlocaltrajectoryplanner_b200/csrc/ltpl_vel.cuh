// ltpl_vel.cuh -- float64 tyre model shared by the brake profiles that stay float64 (k_emergency, k_backup, the opponent
// brake distance of follow mode) and k_export (OTH:941 + LTPL:401-406).  The velocity planner itself is
// ltpl_vel_res.cuh (per-action profiles of a tick) and ltpl_velprofile.cuh (stand-alone solver, BASELINE config 5).
//
// All recurrences are carried in w = v^2: v_next^2 = v^2 + 2 a(v^2) ds needs no sqrt and no division on the dependent
// chain (ay_used = v^2 / radius = w * |kappa|); vx = sqrt(w) and ax = (w1 - w0) / (2 ds) are evaluated afterwards.
#pragma once
#include "ltpl_common.cuh"

// available longitudinal tyre acceleration at w = v^2 on curvature |kappa| (friction ellipse with exponent exp)
// general friction-ellipse exponent: two pow() calls = ~1000 instructions; kept out of line so that the recurrence
// loops of the common exponent 1.0 (LTPL:190 default) stay small in the instruction cache
__device__ __noinline__ double acc_tire_pow(double ratio, double ax_max, double exp_) {
    const double radicand = 1.0 - pow(ratio, exp_);
    return (radicand > 0.0) ? ax_max * pow(radicand, 1.0 / exp_) : 0.0;
}
__device__ __forceinline__ double acc_tire(double w, double kabs, double ax_max, double inv_ay, double exp_) {
    const double ratio = w * kabs * inv_ay;  // ay_used / ay_max, ay_used = v^2 / radius
    if (exp_ == 1.0) {
        const double radicand = 1.0 - ratio;
        return (radicand > 0.0) ? ax_max * radicand : 0.0;
    }
    return acc_tire_pow(ratio, ax_max, exp_);
}

// mode 'decel_forw' with ggv (ax_max, ay_max): -tyre + drag (both negative)
__device__ __forceinline__ double acc_brake(double w, double kabs, double ax_max, double inv_ay, double exp_, double dm) {
    return fma(-w, dm, -acc_tire(w, kabs, ax_max, inv_ay, exp_));
}
// one step of a brake profile (tph.calc_vel_profile_brake) over ds: w_next = w + 2 acc_brake(w) ds, unclamped.  A negative
// value is a negative radicand; what standstill means is left to the caller.
__device__ __forceinline__ double brake_step(double w, double kabs, double ax_max, double inv_ay, double exp_, double dm,
                                             double ds) {
    return fma(2.0 * acc_brake(w, kabs, ax_max, inv_ay, exp_, dm), ds, w);
}

#define LTPL_WARPS_PER_CTA_EXPORT 8

// (P, 7) rows s, x, y, psi, kappa, vx, ax of every kept trajectory, cut to nmbr_export_points (OTH:941, LTPL:401-406)
__global__ void __launch_bounds__(LTPL_WARPS_PER_CTA_EXPORT * 32)
k_export(const __grid_constant__ LtplDims dm, const __grid_constant__ LtplBuffers bf) {
    const int lane = threadIdx.x & 31;
    const int q = sub_path(dm, LTPL_WARPS_PER_CTA_EXPORT);   // a path of this launch's window ...
    if (q < 0) return;
    const int e = bf.traj_row[q];                            // ... and its row of the compact export list
    if (e < 0) return;
    const int n = bf.traj_len[q];
    const int cut = trim_cut(bf, q);   // stateful tick: the trajectory starts at the cut index (OTH:700)
    const PlaneRow<const double> pp = path_row<const double>(bf.path, dm, q, cut);
    const PlaneRow<const double> sv = path_row<const double>(bf.s_vx_ax, dm, q);
    float* out = traj_row(dm, bf, e);
    for (int i = lane; i < n * TRAJ_COLS; i += 32) {   // the points of a row are contiguous
        const int r = i / TRAJ_COLS, col = i - TRAJ_COLS * r;
        double v;
        if (col == TRAJ_S)
            v = sv(SVA_S, r);
        else if (col <= TRAJ_KAPPA)
            v = pp(col - TRAJ_X + PATH_X, r);
        else
            v = sv(col - TRAJ_VX + SVA_VX, r);
        out[i] = (float)v;
    }
}
