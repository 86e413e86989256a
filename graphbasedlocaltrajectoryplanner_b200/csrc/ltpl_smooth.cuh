// ltpl_smooth.cuh -- k_smooth: moving-average smoothing of the velocity profile ([SMOOTHING] filt_window_width > 1).
//
// Reference: every kept trajectory's vx column goes through tph.conv_filt(closed=False) and ax is recomputed from the
// smoothed profile with tph.calc_ax_profile plus the standstill fix-up (OTH:926-941; the brake profile on the backup plan
// the same way, OTH:986-1004).  conv_filt on an open signal of n >= w rows (h = (w - 1) / 2): rows [h, n - h) become the
// mean of vx[i - h .. i + h], the first and the last h rows keep their values; for n < w it is the identity (NumPy
// broadcasts the one-element middle of convolve(.., 'same') into an empty slice).  The filter runs on the WHOLE profile
// before the export cut (LTPL:401-406): exported row 114 depends on rows up to 114 + h.  In a stateful tick the signal is
// vel_course || vx, so the filter crosses the seam.  Row 0 is never changed, so k_emergency (which reads vx[0] and the
// path columns only) and the acceptance test of the velocity kernel are unaffected.
//
// One WARP per path, after the velocity kernel (first tick: it has written the fp32 export rows, so columns 5 and 6 of
// those rows are rewritten here) or after k_prefix (stateful tick: k_export runs behind).  The raw row is staged in shared
// memory before anything is written; sums, ax and the standstill test are float64 in NumPy's operation order.
#pragma once
#include "ltpl_plan.cuh"   // LTPL_WARPS_PER_CTA

__host__ __device__ inline size_t smooth_smem_bytes_per_warp(int p_max) { return sizeof(double) * (size_t)p_max; }

__global__ void __launch_bounds__(LTPL_WARPS_PER_CTA * 32)
k_smooth(const __grid_constant__ LtplDims dm, const __grid_constant__ LtplBuffers bf, const int win, const int export_rows) {
    extern __shared__ __align__(16) unsigned char sm_smem[];
    const int lane = threadIdx.x & 31;
    const int q = sub_path(dm, LTPL_WARPS_PER_CTA);
    if (q < 0) return;
    if (!(bf.status[q] & LTPL_ST_TRAJ_VALID)) return;
    const int B = dm.batch;
    const size_t pplane = (size_t)LTPL_NSLOT * B * dm.p_max;
    const int cut = trim_cut(bf, q);                      // stateful tick: the profile starts at the cut index
    const int n = bf.path_len[q] - cut;                   // rows of the whole profile
    double* raw = reinterpret_cast<double*>(sm_smem) + (size_t)(threadIdx.x >> 5) * dm.p_max;
    const double* S = bf.s_vx_ax + (size_t)q * dm.p_max;
    double* VX = bf.s_vx_ax + pplane + (size_t)q * dm.p_max;
    double* AX = VX + pplane;
    for (int i = lane; i < n; i += 32) raw[i] = VX[i];
    __syncwarp();
    const int h = (win - 1) / 2;
    const bool on = n >= win;
    const double inv_w = 1.0 / (double)win;               // np.ones(w) / float(w)
    // the filtered value of row i: sum of vx[j] * (1 / w), j = i - h .. i + h, left to right (np.convolve)
    auto filt = [&](int i) {
        if (!on || i < h || i >= n - h) return raw[i];
        double acc = 0.0;
        for (int j = i - h; j <= i + h; ++j) acc = __dadd_rn(acc, __dmul_rn(raw[j], inv_w));
        return acc;
    };
    const int e = export_rows ? bf.traj_row[q] : -1;
    const int ne = (e >= 0) ? bf.traj_len[q] : 0;
    float* out = bf.traj + (size_t)max(e, 0) * dm.n_export * 7;
    for (int i = lane; i < n; i += 32) {
        const double v0 = filt(i);
        double a = 0.0;                                   // np.append(ax, [0.0]): the last row
        if (i + 1 < n) {
            const double v1 = filt(i + 1);
            a = (v1 * v1 - v0 * v0) / (2 * (S[i + 1] - S[i]));
            if (fabs(v0) <= 1e-8 && fabs(a) <= 1e-8) a = -5.0;   // np.isclose(vx, 0) & np.isclose(ax, 0) (OTH:939)
        }
        VX[i] = v0;
        AX[i] = a;
        if (i < ne) {
            out[(size_t)i * 7 + 5] = (float)v0;
            out[(size_t)i * 7 + 6] = (float)a;
        }
    }
}
