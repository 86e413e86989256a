// ltpl_stage.cuh -- scenario inputs from device arrays (sm_90a): the host memcpy into pinned staging plus the packed H2D
// copy of a host batch, as one kernel that gathers the caller's device arrays through their strides.
//
// It writes the bytes the host path writes for the same values (BatchPlanner.stage_scenarios / _stage_next), so every
// tick kernel behind it runs exactly as after an upload.
#pragma once
#include "ltpl_common.cuh"

// a 1-, 4- or 8-byte integer of the caller's array as the int32 a NumPy astype(int32) gives (bytes = 1: bool / uint8)
__device__ __forceinline__ int32_t stage_int(const void* p, int64_t i, int bytes) {
    if (bytes == 8) return (int32_t) static_cast<const int64_t*>(p)[i];
    if (bytes == 4) return static_cast<const int32_t*>(p)[i];
    return static_cast<const uint8_t*>(p)[i];
}

// one warp per scenario: lanes strided over the object slots, the prediction points and the n_pred row (coalesced stores
// into the packed input buffer), lane 0 the per-scenario values
__global__ void __launch_bounds__(LTPL_WARPS_PER_CTA * 32)
k_stage(const __grid_constant__ LtplDims dm, const __grid_constant__ LtplBuffers bf, const __grid_constant__ LtplStageSrc src) {
    const int b = blockIdx.x * LTPL_WARPS_PER_CTA + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (b >= dm.batch) return;
    const int K = dm.k_obj, ks = src.k_src;
    double* obj = const_cast<double*>(bf.obj) + (size_t)b * K * 5;
    for (int i = lane; i < K * 5; i += 32) {
        const int k = i / 5, c = i - 5 * k;
        obj[i] = k < ks ? src.obj[b * src.obj_s[0] + k * src.obj_s[1] + c * src.obj_s[2]] : 0.0;
    }
    int32_t* n_pred = const_cast<int32_t*>(bf.n_pred) + (size_t)b * K;
    for (int k = lane; k < K; k += 32)
        n_pred[k] = (src.pred && k < ks) ? src.n_pred[b * src.n_pred_s[0] + k * src.n_pred_s[1]] : -1;
    if (src.kp_dst > 0) {
        const int row = 2 * src.kp_dst;
        double* pred = const_cast<double*>(bf.obj_pred) + (size_t)b * K * row;
        for (int i = lane; i < K * row; i += 32) {
            const int k = i / row, r = i - k * row, p = r >> 1, c = r & 1;
            pred[i] = (src.pred && k < ks && p < src.kp_src)
                          ? src.pred[b * src.pred_s[0] + k * src.pred_s[1] + p * src.pred_s[2] + c * src.pred_s[3]] : 0.0;
        }
    }
    if (lane != 0) return;
    double* pos = const_cast<double*>(bf.pos);
    pos[2 * b] = src.pos[b * src.pos_s[0]];
    pos[2 * b + 1] = src.pos[b * src.pos_s[0] + src.pos_s[1]];
    const double vel = src.vel[b * src.vel_s];
    const_cast<double*>(bf.heading)[b] = src.heading[b * src.heading_s];
    const_cast<double*>(bf.vel)[b] = vel;
    const_cast<double*>(bf.vel_est)[b] = src.vel_est ? src.vel_est[b * src.vel_est_s] : vel;
    const_cast<int32_t*>(bf.n_obj)[b] = src.n_obj[b * src.n_obj_s];
    const_cast<int32_t*>(bf.zone_sel)[b] = src.zone_sel ? src.zone_sel[b * src.zone_sel_s] : -1;
    if (src.sel_action) {
        const_cast<int32_t*>(bf.sel_action)[b] = stage_int(src.sel_action, b * src.sel_action_s, src.sel_action_bytes);
        const_cast<double*>(bf.t_const)[b] = src.t_const ? src.t_const[b * src.t_const_s] : src.t_const_value;
    }
    if (src.restart)
        const_cast<int32_t*>(bf.restart)[b] = stage_int(src.restart, b * src.restart_s, src.restart_bytes) != 0;
    if (src.zone_key_last) {
        // a zone under a NEW id is a new zone object: its unblock window is evaluated at this tick (OLI:155-237)
        const int64_t key = src.zone_key ? src.zone_key[b * src.zone_key_s] : 0;
        if (src.zone_key_rule && key != 0 && key != src.zone_key_last[b]) bf.zone_s0[b] = -1;
        src.zone_key_last[b] = key;
    }
}
