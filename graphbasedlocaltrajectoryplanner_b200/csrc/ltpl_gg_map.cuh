// ltpl_gg_map.cuh -- location dependent friction from a friction map (sm_90a): the gg planes of every path of a scenario
// window, evaluated on the device between the path kernel and the velocity kernel.
//
// A tick with buffers.gg_map gives what calc_vel_profile(local_gg={action: [map(path[:, 0:2])]}) gives with the planes
// set by the caller (OTH:649-666): the planes are the only thing the map changes, so k_vel_res<.., GG>, k_emergency and
// k_backup read them exactly as they read uploaded planes.
#pragma once
#include "ltpl_common.cuh"

// bilinear interpolation of the four vertices around (x, y), clamped to the grid, in one fixed operation order without
// FMA (tests/gg_map_ref.py restates it in NumPy; the planes equal that restatement bit for bit):
//   u = (x - x0) * inv_cell, clamped to [0, nx - 1];  i = min(floor(u), nx - 2);  tx = u - i   (v, j, ty likewise)
//   a = (1 - ty) * ((1 - tx) * g[j][i] + tx * g[j][i+1]) + ty * ((1 - tx) * g[j+1][i] + tx * g[j+1][i+1])
__device__ __forceinline__ double2 gg_map_at(const LtplParams& prm, const double2* __restrict__ map, double x, double y) {
    const double u = fmin(fmax(__dmul_rn(__dsub_rn(x, prm.gg_map_x0), prm.gg_map_inv_cell), 0.0), (double)(prm.gg_map_nx - 1));
    const double v = fmin(fmax(__dmul_rn(__dsub_rn(y, prm.gg_map_y0), prm.gg_map_inv_cell), 0.0), (double)(prm.gg_map_ny - 1));
    const int i = min((int)floor(u), prm.gg_map_nx - 2), j = min((int)floor(v), prm.gg_map_ny - 2);
    const double tx = __dsub_rn(u, (double)i), ty = __dsub_rn(v, (double)j);
    const double sx = __dsub_rn(1.0, tx), sy = __dsub_rn(1.0, ty);
    const size_t r0 = (size_t)j * prm.gg_map_nx + i, r1 = r0 + prm.gg_map_nx;
    const double2 g00 = __ldg(map + r0), g01 = __ldg(map + r0 + 1), g10 = __ldg(map + r1), g11 = __ldg(map + r1 + 1);
    double2 a;
    a.x = __dadd_rn(__dmul_rn(sy, __dadd_rn(__dmul_rn(sx, g00.x), __dmul_rn(tx, g01.x))),
                    __dmul_rn(ty, __dadd_rn(__dmul_rn(sx, g10.x), __dmul_rn(tx, g11.x))));
    a.y = __dadd_rn(__dmul_rn(sy, __dadd_rn(__dmul_rn(sx, g00.y), __dmul_rn(tx, g01.y))),
                    __dmul_rn(ty, __dadd_rn(__dmul_rn(sx, g10.y), __dmul_rn(tx, g11.y))));
    return a;
}

// one warp per path q = slot * B + b of the window, lanes strided over its points [0, path_len): coalesced x / y loads
// and gg stores, four 16-byte corner gathers per point.  Points behind path_len are left as they are.
__global__ void __launch_bounds__(LTPL_WARPS_PER_CTA * 32)
k_gg_map(const __grid_constant__ LtplParams prm, const __grid_constant__ LtplDims dm, const __grid_constant__ LtplBuffers bf) {
    const int q = sub_path(dm, LTPL_WARPS_PER_CTA);
    if (q < 0) return;
    const int n = bf.path_len[q];
    const PlaneRow<const double> path = path_row<const double>(bf.path, dm, q);
    const PlaneRow<double> gg = path_row(bf.gg, dm, q);
    const double2* map = reinterpret_cast<const double2*>(bf.gg_map);
    for (int i = threadIdx.x & 31; i < n; i += 32) {
        const double2 a = gg_map_at(prm, map, path(PATH_X, i), path(PATH_Y, i));
        gg(GG_AX, i) = a.x;
        gg(GG_AY, i) = a.y;
    }
}
