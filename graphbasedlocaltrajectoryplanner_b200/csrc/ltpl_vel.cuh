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

#define LTPL_WARPS_PER_CTA_EXPORT 8

// (P, 7) rows s, x, y, psi, kappa, vx, ax of every kept trajectory, cut to nmbr_export_points (OTH:941, LTPL:401-406)
__global__ void __launch_bounds__(LTPL_WARPS_PER_CTA_EXPORT * 32)
k_export(const __grid_constant__ LtplDims dm, const __grid_constant__ LtplBuffers bf) {
    const int B = dm.batch;
    const int lane = threadIdx.x & 31;
    const int q = sub_path(dm, LTPL_WARPS_PER_CTA_EXPORT);   // a path of this launch's window ...
    if (q < 0) return;
    const int e = bf.traj_row[q];                            // ... and its row of the compact export list
    if (e < 0) return;
    const int n = bf.traj_len[q];
    const size_t pplane = (size_t)LTPL_NSLOT * B * dm.p_max;
    const int cut = bf.trim ? bf.trim[4 * q + 2] : 0;   // stateful tick: the trajectory starts at the cut index (OTH:700)
    const double* pp = bf.path + (size_t)q * dm.p_max + cut;
    const double* sv = bf.s_vx_ax + (size_t)q * dm.p_max;
    float* out = bf.traj + (size_t)e * dm.n_export * 7;
    for (int i = lane; i < n * 7; i += 32) {
        const int r = i / 7, col = i - 7 * r;
        double v;
        if (col == 0)
            v = sv[r];
        else if (col <= 4)
            v = pp[(size_t)(col - 1) * pplane + r];
        else
            v = sv[(size_t)(col - 4) * pplane + r];
        out[i] = (float)v;
    }
}
