// ltpl_select.cuh -- the trajectory each scenario takes (sm_90a): the first action of a preference list that the last
// velocity call returned, and a dense copy of its export row (ltpl_select_batch).
//
// The reference's loops pick one trajectory after every tick, the first action of a preference order that the returned
// set contains (main_min_example.py:83-85, main_std_example.py:101-103).  This kernel applies that rule to the result
// buffers exactly as the tick left them:
//   - a slot action a is returned when some slot s has action_id[s][b] == a and traj_row[s][b] >= 0 (the trajectory
//     keys of the reference's dict);
//   - 'emergency' is returned when the velocity call ran with params.incl_emerg_traj, some slot trajectory was kept
//     and em_info[b][0] >= 0 (OTH:1027-1034).  em_info alone is not trusted: a buffer set without memory keeps the
//     values of an earlier call that had the emergency trajectory.
#pragma once
#include "ltpl_common.cuh"

// an entry of a preference list as a 64-bit value, so that no wider integer wraps onto an action id
__device__ __forceinline__ int64_t select_entry(const void* p, int64_t i, int bytes) {
    if (bytes == 8) return static_cast<const int64_t*>(p)[i];
    if (bytes == 4) return static_cast<const int32_t*>(p)[i];
    return static_cast<const int8_t*>(p)[i];
}

// one warp per scenario: lane 0 resolves the pick (at most LTPL_SELECT_MAX entries x NSLOT slots + emergency), then the
// warp copies the selected export row (n_export x 7 floats) to sel_traj[b], zeros where nothing was selected.  `emerg`:
// params.incl_emerg_traj of the velocity call that wrote the buffers.
__global__ void __launch_bounds__(LTPL_WARPS_PER_CTA * 32)
k_select(const __grid_constant__ LtplDims dm, const __grid_constant__ LtplBuffers bf, const __grid_constant__ LtplSelect sel,
         const int emerg) {
    const int b = blockIdx.x * LTPL_WARPS_PER_CTA + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (b >= dm.batch) return;
    const int B = dm.batch;
    int row = -1;
    if (lane == 0) {
        int act = LTPL_ACT_NONE, len = 0, id = -1;
        bool kept = false;
        for (int s = 0; s < LTPL_NSLOT; ++s) kept |= bf.traj_row[s * B + b] >= 0;
        for (int i = 0; i < sel.prefer_len && act == LTPL_ACT_NONE; ++i) {
            const int64_t a = select_entry(sel.prefer, b * sel.prefer_s[0] + i * sel.prefer_s[1], sel.prefer_bytes);
            if (a == LTPL_ACT_EMERGENCY) {
                if (emerg && kept && bf.em_info[3 * b] >= 0) {
                    act = LTPL_ACT_EMERGENCY;
                    row = bf.em_info[3 * b];
                    len = bf.em_info[3 * b + 1];
                    id = bf.em_info[3 * b + 2];
                }
            } else if (a >= 0 && a < LTPL_ACT_EMERGENCY) {
                for (int s = 0; s < LTPL_NSLOT; ++s) {   // 'straight' and 'follow' share slot 0: match the id, not the slot
                    const int q = s * B + b;
                    if (bf.action_id[q] == a && bf.traj_row[q] >= 0) {
                        act = (int)a;
                        row = bf.traj_row[q];
                        len = bf.traj_len[q];
                        id = bf.traj_id[q];
                        break;
                    }
                }
            }
        }
        sel.sel_action[b * sel.sel_action_s] = act;
        int32_t* info = sel.sel_info + 4 * (size_t)b;
        info[0] = act;
        info[1] = row;
        info[2] = len;
        info[3] = id;
    }
    if (!sel.sel_traj) return;
    row = __shfl_sync(0xffffffffu, row, 0);
    // a row is n_export * 7 floats: 16-byte aligned only when n_export % 4 == 0 (115 rows: 4-byte aligned)
    const int n = dm.n_export * 7;
    float* __restrict__ dst = sel.sel_traj + (size_t)b * n;
    const float* __restrict__ src = row >= 0 ? bf.traj + (size_t)row * n : nullptr;
    const bool wide = (n & 3) == 0 && (reinterpret_cast<uintptr_t>(bf.traj) & 15) == 0 &&
                      (reinterpret_cast<uintptr_t>(sel.sel_traj) & 15) == 0;
    if (wide) {
        float4* __restrict__ d4 = reinterpret_cast<float4*>(dst);
        const float4* __restrict__ s4 = reinterpret_cast<const float4*>(src);
#pragma unroll 4
        for (int i = lane; i < (n >> 2); i += 32) d4[i] = src ? s4[i] : make_float4(0.f, 0.f, 0.f, 0.f);
    } else {
#pragma unroll 4
        for (int i = lane; i < n; i += 32) dst[i] = src ? src[i] : 0.f;
    }
}
