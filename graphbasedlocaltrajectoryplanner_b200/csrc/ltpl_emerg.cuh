// ltpl_emerg.cuh -- k_emergency: the 'emergency' entry of the trajectory set (calc_vel_profile(incl_emerg_traj=True)).
//
// Reference: OTH:1027-1034 picks the FIRST key of the kept trajectory dict (slot order follow|straight, left, right) and
// calls calc_brake_emergency (helper_funcs/src/calc_brake_emergency.py:9-47): tph.calc_vel_profile_brake along that
// trajectory (kappa = column 4, el = diff(s), v_start = vx[0], drag 0.854, mass 1160, loc_gg = the caller's local_gg
// WITHOUT gg_scale, friction-ellipse exponent 1.0) and tph.calc_ax_profile(eq_length_output=True); the result keeps
// s, x, y, psi, kappa of the base trajectory, shares its id and is cut to nmbr_export_points rows like every other
// trajectory (LTPL:401-406).
//
// One WARP per scenario, launched after k_export: lanes stage s and kappa of the first n_export + 1 points in shared
// memory, lane 0 runs the brake recurrence in w = v^2 (same arithmetic as brake_profile_w), all lanes write the fp32 row
// into the next free row of the compact export buffer (queue_cnt[2]); the f64 velocities also go to em_vx (stateful ticks:
// get_ref_idx reads them when the caller executes this trajectory, OTH:307-309 / 518-601).
#pragma once
#include "ltpl_vel.cuh"

#define LTPL_EM_DRAG 0.854   // calc_brake_emergency.py:6
#define LTPL_EM_MASS 1160.0  // calc_brake_emergency.py:5

__host__ __device__ inline size_t emerg_smem_bytes_per_warp(int n_export) {
    return sizeof(double) * 3 * (size_t)(n_export + 1);
}

__global__ void __launch_bounds__(LTPL_WARPS_PER_CTA * 32)
k_emergency(const __grid_constant__ LtplParams prm, const __grid_constant__ LtplDims dm, const __grid_constant__ LtplBuffers bf) {
    extern __shared__ __align__(16) unsigned char em_smem[];
    const int lane = threadIdx.x & 31;
    const int wib = threadIdx.x >> 5;
    const int b = sub_scenario(dm, LTPL_WARPS_PER_CTA);
    if (b < 0) return;
    const int B = dm.batch;
    int* info = bf.em_info + 3 * (size_t)b;
    int q = -1;
    for (int s = LTPL_NSLOT - 1; s >= 0; --s)
        if (bf.traj_len[s * B + b] > 0) q = s * B + b;
    if (q < 0) {
        if (lane == 0) {
            info[0] = -1;
            info[1] = 0;
            info[2] = -1;
        }
        return;
    }
    const int cut = bf.trim ? bf.trim[4 * q + 2] : 0;   // stateful tick: the trajectory starts at the cut index
    const int n = bf.path_len[q] - cut;
    const int ne = min(n, dm.n_export);          // exported rows
    const int m = min(n, ne + 1);                // points the rows depend on (ax of row ne - 1 needs w[ne])
    double* ss = reinterpret_cast<double*>(em_smem) + (size_t)wib * 3 * (dm.n_export + 1);
    double* sk = ss + (dm.n_export + 1);
    double* sw = sk + (dm.n_export + 1);
    const size_t pplane = (size_t)LTPL_NSLOT * B * dm.p_max;
    const double* s_row = bf.s_vx_ax + (size_t)q * dm.p_max;
    const double* vx_row = s_row + pplane;
    const double* pp = bf.path + (size_t)q * dm.p_max + cut;
    for (int i = lane; i < m; i += 32) {
        ss[i] = s_row[i];
        sk[i] = fabs(pp[3 * pplane + i]);
    }
    __syncwarp();
    if (lane == 0) {
        const double dmq = LTPL_EM_DRAG / LTPL_EM_MASS;
        const double inv_ay = 1.0 / prm.gg_ay;
        // location dependent local_gg: the rows of the base trajectory, cut at its start (action_set_path_param_gg, OTH:1030)
        const double* ggr = bf.gg ? bf.gg + (size_t)q * dm.p_max + cut : nullptr;
        double v0 = vx_row[0];
        if (v0 < 0.0) v0 = 0.0;
        double w = v0 * v0;
        bool stopped = false;
        sw[0] = w;
        #pragma unroll 1
        for (int i = 0; i + 1 < m; ++i) {
            if (!stopped) {
                const double a = ggr ? acc_brake(w, sk[i], ggr[i], 1.0 / ggr[pplane + i], 1.0, dmq)
                                     : acc_brake(w, sk[i], prm.gg_ax, inv_ay, 1.0, dmq);
                const double nx = fma(2.0 * a, ss[i + 1] - ss[i], w);
                if (nx < 0.0) {   // tph.calc_vel_profile_brake: negative radicand -> the rest of the profile stays 0
                    stopped = true;
                    w = 0.0;
                } else {
                    w = nx;
                }
            }
            sw[i + 1] = w;
        }
    }
    __syncwarp();
    int row = 0;
    if (lane == 0) row = atomicAdd(&bf.queue_cnt[2], 1);
    row = __shfl_sync(LTPL_FULL, row, 0);
    float* out = bf.traj + (size_t)row * dm.n_export * 7;
    for (int i = lane; i < ne; i += 32) {
        double a = 0.0;                          // eq_length_output: the last point of the FULL profile gets 0
        if (i + 1 < n) a = (sw[i + 1] - sw[i]) / (2 * (ss[i + 1] - ss[i]));
        float* o = out + (size_t)i * 7;
        o[0] = (float)ss[i];
        o[1] = (float)pp[0 * pplane + i];
        o[2] = (float)pp[1 * pplane + i];
        o[3] = (float)pp[2 * pplane + i];
        o[4] = (float)pp[3 * pplane + i];
        const double v = sqrt(sw[i]);
        o[5] = (float)v;
        if (bf.em_vx) bf.em_vx[(size_t)b * dm.n_export + i] = v;   // f64 copy: memory of an executed 'emergency' (k_ref)
        o[6] = (float)a;
    }
    if (lane == 0) {
        info[0] = row;
        info[1] = ne;
        info[2] = bf.traj_id[q];
    }
}
