// ltpl_traj_base.cuh -- trajectory ids from a device counter (sm_90a), for ticks replayed from a CUDA graph.
//
// A captured tick keeps the params it was captured with, so params.traj_base_id (+10 per velocity call, OTH:669) would
// repeat the captured tick's ids on every replay.  With buffers.traj_base the velocity kernels run with traj_base_id = 0
// (ids = action id) and this kernel, behind the window join, adds the next base from the counter: the bytes of the same
// call with traj_base_id = that base.
//
// Which ids this call wrote: with base 0 they are the action ids, 0 .. 9, while every id of an earlier call already has
// its base >= 10 (the counter is >= 0 and advances by 10 before use; an eager call's base is 10 per call).  So exactly
// the ids in [0, 10) get the base.  An id the velocity stage left as it was -- a path a repeated velocity call without
// calc_paths rejects after an earlier call accepted it -- keeps its old value, as in the eager call.
#pragma once
#include "ltpl_common.cuh"

#define LTPL_TRAJ_BASE_THREADS 1024

// ONE CTA: every thread reads the counter, the block barrier orders those reads before thread 0 writes counter + 10.
// A single CTA needs neither a second launch nor a ticket word beside the counter, and the work is small: 4 ints per
// scenario (NSLOT ids + one emergency id), 40 000 at 10 000 scenarios.  em_info: NULL unless the call wrote emergency
// trajectories (params.incl_emerg_traj); otherwise nothing wrote it and it is left alone.
__global__ void __launch_bounds__(LTPL_TRAJ_BASE_THREADS)
k_traj_base(int32_t* traj_base, int32_t* __restrict__ traj_id, int32_t* __restrict__ em_info, const int n_ids,
            const int batch) {
    const int32_t base = *traj_base + 10;
    __syncthreads();
    if (threadIdx.x == 0) *traj_base = base;
    for (int i = threadIdx.x; i < n_ids; i += LTPL_TRAJ_BASE_THREADS) {
        const int32_t v = traj_id[i];
        if (v >= 0 && v < 10) traj_id[i] = v + base;
    }
    if (em_info)
        for (int b = threadIdx.x; b < batch; b += LTPL_TRAJ_BASE_THREADS) {
            const int32_t v = em_info[3 * b + 2];
            if (em_info[3 * b] >= 0 && v >= 0 && v < 10) em_info[3 * b + 2] = v + base;
        }
}
