// ltpl_vel_res.cuh -- k_vel_res: OTH.calc_vel_profile per action (OTH:688-1025) with every path RESIDENT in shared memory.
//
// The velocity solver (tph.calc_vel_profile, restated in oracle/tph_port.py:463-538) is a serial recurrence per path and
// a 10 k-scenario batch only holds ~13 k paths: the kernel is bound by (steps on the critical chain of one path) x
// (dependent-issue latency of one step).  Design:
//   * one CTA = 2 warps = VR_P queued paths of one class (follow / other).  The kappa and el rows of all its paths arrive
//     with ONE round of TMA bulk copies (cp.async.bulk + mbarrier: 2 copies per path, all in flight together) and are
//     compacted in place to fp32 K' = |kappa| / ay_max and E2 = 2 el; every later access of the recurrences is a
//     shared-memory access of 29 cycles instead of an L2 round trip, no intermediate profile ever leaves the SM.
//     Per path and point: K', E2, W (complete profile), SRC (brake / control profile), S (arc length) = 20 bytes.
//   * the recurrences run in fp32 (BASELINE.json north_star: "fp32 elementwise for ... velocity integration"), in
//     w = v^2 (no sqrt / division on the chain except the machine-limit lookup), one LANE per path.  Accumulated
//     rounding over a 300-point path is < 1e-6 relative in w (tests: 1e-4).  Arc lengths, s-coordinate searches and
//     every index decision on them stay float64.
//   * follow paths: warp 0 runs the complete profile (lanes 0..P-1) and, in the same instruction stream, the ego brake
//     profile (lanes P..2P-1), then the backward sweep of the complete profile; warp 1 meanwhile matches the opponent
//     (brake distance on the global race line, nearest path points), then -- behind a named barrier -- derives the
//     follow scalars (CVPF:139-247) and runs the control profile forward / backward.  Two warps = the two independent
//     dependency chains of CVPF:263-310 advance concurrently.
//   * the element-wise end (min of profiles, vx = sqrt(w), ax, standstill fix-up, OTH:926-941) runs on all 64 threads
//     with coalesced float64 stores into the s / vx / ax planes.
#pragma once
#include "ltpl_vel.cuh"

#ifndef VR_P
#define VR_P 8                       // paths per CTA (<= 16: the brake chain shares warp 0 with the complete profile)
#endif
#define VR_THREADS 64
#define VR_MAXM 16                   // points per lane in the arc-length scan: nmax <= 32 * VR_MAXM = 512

// per path and point: E2, W, K', SRC, S (+ AX, IAY: longitudinal tyre limit and 1 / lateral limit per point when a location
// dependent local_gg is given)
__host__ __device__ inline size_t vr_smem_bytes(int nmax, bool gg) {
    return (size_t)VR_P * (gg ? 7 : 5) * nmax * sizeof(float);
}

// ---- TMA bulk copy + mbarrier (PTX) ---------------------------------------------------------------------------------
__device__ __forceinline__ unsigned vr_s32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void vr_mbar_init(unsigned long long* bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(vr_s32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void vr_mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(vr_s32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void vr_bulk_g2s(void* dst, const void* src, unsigned bytes, unsigned long long* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     vr_s32(dst)),
                 "l"(src), "r"(bytes), "r"(vr_s32(bar))
                 : "memory");
}
__device__ __forceinline__ void vr_mbar_wait(unsigned long long* bar, unsigned parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "VR_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra VR_DONE;\n"
        "bra VR_WAIT;\n"
        "VR_DONE:\n"
        "}\n" ::"r"(vr_s32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void vr_bar_arrive(int id) {
    __threadfence_block();
    asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(VR_THREADS) : "memory");
}
__device__ __forceinline__ void vr_bar_sync(int id) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(VR_THREADS) : "memory");
}

// ---- fp32 recurrences -----------------------------------------------------------------------------------------------
// machine table (np.interp(v, ax_max_machines[:, 0], ax_max_machines[:, 1])) as n + 1 segments in shared memory:
//   segment 0: v < xp[0] -> fp[0];  segment k = 1 .. n-1: [xp[k-1], xp[k]) linear;  segment n: v >= xp[n-1] -> fp[n-1]
#define VR_TAB (LTPL_MAX_AXM + 2)
struct VRCfg {
    float ax_max, dm, exp_, inv_exp;
    const float* xl;   // [n + 2] lower bounds of the segments, xl[0] = -inf, xl[n + 1] = +inf
    const float* x0;   // [n + 1] abscissa the segment's line is anchored at
    const float* f0;   // [n + 1]
    const float* sl;   // [n + 1] slopes exactly as np.interp forms them (0 on the two outer segments)
    int n_seg;         // n + 1
};
__device__ __forceinline__ void vr_stage_axm(const LtplParams& prm, float* s_tab /* [4 * VR_TAB] shared */) {
    const int n = prm.n_axm;
    for (int k = threadIdx.x; k <= n + 1; k += blockDim.x) {
        s_tab[k] = (k == 0) ? -CUDART_INF_F : ((k == n + 1) ? CUDART_INF_F : (float)prm.axm_v[k - 1]);
        if (k <= n) {
            const bool outer = (k == 0 || k == n);
            s_tab[VR_TAB + k] = outer ? 0.0f : (float)prm.axm_v[k - 1];
            s_tab[2 * VR_TAB + k] = (k == 0) ? (float)prm.axm_a[0] : (float)prm.axm_a[k - 1];
            s_tab[3 * VR_TAB + k] = outer ? 0.0f : (float)prm.axm_s[k - 1];
        }
    }
}
__device__ __forceinline__ VRCfg vr_make_cfg(const LtplParams& prm, const float* s_tab) {
    VRCfg c;
    c.ax_max = (float)(prm.gg_ax * prm.gg_scale);
    c.dm = (float)(prm.drag_coeff / prm.m_veh);
    c.exp_ = (float)prm.dyn_model_exp;
    c.inv_exp = (float)(1.0 / prm.dyn_model_exp);
    c.xl = s_tab;
    c.x0 = s_tab + VR_TAB;
    c.f0 = s_tab + 2 * VR_TAB;
    c.sl = s_tab + 3 * VR_TAB;
    c.n_seg = prm.n_axm + 1;
    return c;
}
__device__ __forceinline__ float vr_rcp(float x) {   // 1 / x, one MUFU (no IEEE fix-up code on the chain); 1 / 0 = +inf
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float vr_sqrt(float x) {
    float y;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
// friction ellipse with a general exponent: two powf calls; out of line (the default exponent 1.0 never gets here)
__device__ __noinline__ float vr_tire_pow(float ratio, float ax_max, float e, float inv_e) {
    const float rad = 1.0f - powf(ratio, e);
    return (rad > 0.0f) ? ax_max * powf(rad, inv_e) : 0.0f;
}
// available longitudinal tyre acceleration at w = v^2 with K = |kappa| / ay_max (tph.calc_ax_poss)
// ax: ax_max of the point (location dependent local_gg, OTH:649-666) or the constant c.ax_max
template <bool EXP1>
__device__ __forceinline__ float vr_tire(const VRCfg& c, float w, float K, float ax) {
    if (EXP1) return ax * fmaxf(fmaf(-w, K, 1.0f), 0.0f);
    return vr_tire_pow(w * K, ax, c.exp_, c.inv_exp);
}

// Forward sweep of one lane's profile on points [lo, hi] of its path (K, E2, W: the path's shared-memory rows):
// tph.__solver_fb_acc_profile(backwards=False): start value min(curvature limit, wcap), acceleration phases from the
// rising edges of the curvature-limit profile, end clamp we (< 0: none).  The step is branch-free (selects).  The
// machine limit is a table segment cached in registers; v moves slowly, and when a lane leaves its segment the WHOLE
// warp takes one step to the neighbouring segment (warp-uniform branch: a miss never serialises lanes).
// (pure brake profiles: vr_brake below)
// GG: per-point longitudinal tyre limit AX[] (location dependent local_gg), else the constant c.ax_max
template <bool EXP1, bool GG>
__device__ __noinline__ void vr_forward(const VRCfg c, bool on, const float* __restrict__ K,
                                        const float* __restrict__ E2, const float* __restrict__ AX, float* __restrict__ W,
                                        int lo, int hi, float wcap, float we, float wmax, int nmax) {
    const int len = (on && hi >= lo) ? hi - lo : -1;
    int lmax = len;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) lmax = max(lmax, __shfl_xor_sync(LTPL_FULL, lmax, o));
    if (lmax < 0) return;
    if (len < 0) lo = 0;
    float k_prev = K[lo], ax_prev = GG ? AX[lo] : c.ax_max;
    float cur = fminf(fminf(vr_rcp(k_prev), wmax), wcap);
    if (len >= 0) W[lo] = cur;
    float o_prev = cur;
    bool prev_rise = false, active = false;
    int sg = 1;   // cached table segment
    float xlo = c.xl[1], xhi = c.xl[2], x0 = c.x0[1], f0 = c.f0[1], sl = c.sl[1];
    // lanes whose profile has ended keep stepping on clamped indices without storing: no select in the step needs `live`
    const int pcap = nmax - 1;
#pragma unroll 2
    for (int i = 1; i <= lmax; ++i) {
        const bool live = i <= len;
        const int p = min(lo + i, pcap);
        const float kq = K[p], e2 = E2[p - 1];
        const float o_n = fminf(vr_rcp(kq), wmax);
        const bool rise = o_n > o_prev;
        active = active || (rise && !prev_rise);
        const float v = vr_sqrt(fmaxf(cur, 0.0f));
        const bool need = live && active;   // machine limit: only inside an acceleration phase
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
        const float a_t = vr_tire<EXP1>(c, cur, k_prev, ax_prev);
        const float a_m = fmaf(sl, v - x0, f0);                              // mode 'accel_forw': min(tyre, machine(v))
        const float a = fmaf(-cur, c.dm, fminf(a_t, a_m));                   // + drag
        const float wn = fmaf(a, e2, cur);
        const float nxt = active ? fminf(wn, o_n) : o_n;
        active = active && !(wn > wmax);
        if (live) W[p] = nxt;
        cur = nxt;
        prev_rise = rise;
        o_prev = o_n;
        k_prev = kq;
        if (GG) ax_prev = AX[p];
    }
    if (len >= 0 && we >= 0.0f && W[hi] > we) W[hi] = we;
}
// Forward sweep of a pure brake profile (tph.calc_vel_profile_brake, mode 'decel_forw': -tyre + drag from wcap on): the
// step of vr_forward for a brake lane without everything a brake lane does not use (curvature cap, acceleration phases,
// machine limit and its sqrt / vote) -- same arithmetic, shorter chain.
template <bool EXP1, bool GG>
__device__ __noinline__ void vr_brake(const VRCfg c, bool on, const float* __restrict__ K, const float* __restrict__ E2,
                                      const float* __restrict__ AX, float* __restrict__ W, int lo, int hi, float wcap,
                                      float we, int nmax) {
    const int len = (on && hi >= lo) ? hi - lo : -1;
    int lmax = len;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) lmax = max(lmax, __shfl_xor_sync(LTPL_FULL, lmax, o));
    if (lmax < 0) return;
    if (len < 0) lo = 0;
    float k_prev = K[lo], ax_prev = GG ? AX[lo] : c.ax_max;
    float cur = wcap;
    // A brake profile approaches w = 0 from large values: the absolute rounding of an fp32 accumulator (1e-3 after 100
    // steps from 60 m/s) would be several mm/s in v just before standstill.  It therefore ACCUMULATES in float64 (the
    // acceleration itself stays fp32: its error enters scaled by the step).
    double cur64 = (double)cur;
    if (len >= 0) W[lo] = cur;
    const int pcap = nmax - 1;
#pragma unroll 2
    for (int i = 1; i <= lmax; ++i) {
        const int p = min(lo + i, pcap);
        const float kq = K[p], e2 = E2[p - 1];
        const float a = fmaf(-cur, c.dm, -vr_tire<EXP1>(c, cur, k_prev, ax_prev));
        cur64 = fmax(cur64 + (double)a * (double)e2, 0.0);   // negative radicand: standstill, the rest stays 0
        cur = (float)cur64;
        if (i <= len) W[p] = cur;
        k_prev = kq;
        if (GG) ax_prev = AX[p];
    }
    if (len >= 0 && we >= 0.0f && W[hi] > we) W[hi] = we;
}
// Backward sweep (flipped arrays, mode 'decel_backw', one look-ahead correction); returns w[lo] afterwards.
// GG (location dependent local_gg): tph flips radii, el_lengths and the profile for this sweep but NOT the per-point ggv
// (oracle/tph_port.py:463-538: p_ggv[i] is indexed with the flipped counter), so the point p of the profile [lo, hi] takes
// the tyre limits of its mirror point lo + hi - p -- reproduced here: K'(p) = |kappa(p)| / ay(mirror), ax(mirror).
template <bool EXP1, bool GG>
__device__ __noinline__ float vr_backward(const VRCfg c, bool on, const float* __restrict__ K,
                                          const float* __restrict__ E2, const float* __restrict__ AX,
                                          const float* __restrict__ IAY, float* __restrict__ W, int lo, int hi,
                                          float wmax) {
    float cur = 0.0f;
    if (on && hi >= lo) {
        cur = W[hi];
        const int mir = lo + hi;
        float o_prev = cur;
        float k_p = GG ? K[hi] * vr_rcp(IAY[hi]) * IAY[mir - hi] : K[hi];
        float ax_p = GG ? AX[mir - hi] : c.ax_max;
        bool prev_rise = false, active = false;
#pragma unroll 2
        for (int p = hi - 1; p >= lo; --p) {
            const float o_n = W[p], e2 = E2[p];
            const float kq = GG ? K[p] * vr_rcp(IAY[p]) * IAY[mir - p] : K[p];
            const float axq = GG ? AX[mir - p] : c.ax_max;
            const bool rise = o_n > o_prev;
            active = active || (rise && !prev_rise);
            const float a = fmaf(cur, c.dm, vr_tire<EXP1>(c, cur, k_p, ax_p));
            float wn = fmaf(a, e2, cur);
            const float a2 = fmaf(wn, c.dm, vr_tire<EXP1>(c, wn, kq, axq));
            const float wt = fmaf(a2, e2, cur);
            wn = fminf(wn, wt);
            const float nxt = active ? fminf(wn, o_n) : o_n;
            active = active && !(wn > wmax);
            W[p] = nxt;
            cur = nxt;
            prev_rise = rise;
            o_prev = o_n;
            k_p = kq;
            ax_p = axq;
        }
    }
    return cur;
}

// first index i in [0, n) with s[i] >= thr (s non-decreasing), n if none: located on the fp32 copy in shared memory,
// decided on the float64 values in global memory (rounding to fp32 is monotone, so the answer is never in front of the
// fp32 candidate and at most a few entries behind it)
__device__ __forceinline__ int vr_first_ge_s(const float* __restrict__ S32, const double* __restrict__ sg, int n,
                                             double thr) {
    const float t = (float)thr;
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (S32[mid] >= t)
            hi = mid;
        else
            lo = mid + 1;
    }
    while (lo < n && __ldcg(sg + lo) < thr) ++lo;
    return lo;
}
// first index i in [0, n) with W[i] <= thr (W non-increasing), n if none
__device__ __forceinline__ int vr_first_le(const float* __restrict__ W, int n, float thr) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (W[mid] <= thr)
            hi = mid;
        else
            lo = mid + 1;
    }
    return lo;
}

// get_s_coord.py:8-99 on an open polyline once the nearest index nb is known (x, y, el: rows of the path planes, sg: the
// float64 arc lengths of the path)
__device__ __forceinline__ double vr_s_coord_from_nb(const double* x, const double* y, const double* el, const double* sg,
                                                     int n, int nb, double px, double py) {
    const int idx1 = max(nb - 1, 0), idx2 = min(nb + 1, n - 1);
    const double xn = x[nb], yn = y[nb];
    int ia, ib;
    if (angle_cmp(make_double2(xn, yn), px, py, make_double2(x[idx1], y[idx1]), make_double2(x[idx2], y[idx2])).gt) {
        ia = idx1;
        ib = nb;
    } else {
        ia = nb;
        ib = idx2;
    }
    const bool ins = el[0] > 0.05;   // leading 0 inserted into s_array = cumsum(el) (get_s_coord.py:67-68)
    const double s_ia = __ldcg(sg + ia);
    const double sbase = ins ? s_ia : __dadd_rn(s_ia, el[ia]);
    const double ax = x[ia], ay = y[ia], bx = x[ib] - ax, by = y[ib] - ay;
    const double t = __ddiv_rn(__dadd_rn(__dmul_rn(px - ax, bx), __dmul_rn(py - ay, by)), __dadd_rn(sq_rn(bx), sq_rn(by)));
    const double sx = __dadd_rn(ax, __dmul_rn(t, bx)), sy = __dadd_rn(ay, __dmul_rn(t, by));
    const double ds = sqrt(__dadd_rn(sq_rn(ax - sx), sq_rn(ay - sy)));
    return __dadd_rn(sbase, ds);
}

// kappa row (float64, staged at X2 | X3 with `sh` leading junk elements) -> K' (fp32) in place at X2: batches of 32
// points in ascending order; a batch's writes only cover sources of earlier batches
// gg_row: the path's rows of the local_gg planes (ax at gg_row, ay at gg_row + gg_plane; NULL: constant local_gg): K' uses
// the lateral limit of its point, AX gets the longitudinal one (both times gg_scale, VPFB:213-214)
__device__ __forceinline__ void vr_convert_kappa(float* X2, float* AX, float* IAY, int n, int sh, double inv_ay,
                                                 const double* gg_row, size_t gg_plane, double gg_scale, int lane) {
    const double* src = reinterpret_cast<const double*>(X2) + sh;
#pragma unroll 1
    for (int p0 = 0; p0 < n; p0 += 32) {
        const int p = p0 + lane;
        const double k = (p < n) ? src[p] : 0.0;
        double iay = inv_ay;
        if (gg_row && p < n) {
            iay = 1.0 / (gg_row[gg_plane + p] * gg_scale);
            AX[p] = (float)(gg_row[p] * gg_scale);
            IAY[p] = (float)iay;
        }
        __syncwarp();
        if (p < n) X2[p] = (float)(fabs(k) * iay);
    }
    __syncwarp();
}
// el row (float64, staged at X0 | X1) -> E2 = 2 el (fp32) in place at X0, arc lengths s = [0, cumsum(el[:-1])] (OTH:743)
// as float64 into the s plane and as fp32 into X4.  Rounds of VR_SC chunks of 32 points: lane l owns the points l,
// l + 32, ... of a round (coalesced), every chunk is one warp scan and the VR_SC scans of a round are independent
// instruction streams (ILP).  In place: a round's writes (4 bytes per point) only cover sources (8 bytes per point) of
// this and earlier rounds, and a round reads all its sources before it writes.
#define VR_SC 6
__device__ __forceinline__ void vr_convert_el(float* X0, float* X4, double* s_out, int n, int sh, int lane) {
    const double* src = reinterpret_cast<const double*>(X0) + sh;
    double base = 0.0;
#pragma unroll 1
    for (int c0 = 0; c0 < n; c0 += 32 * VR_SC) {
        double e[VR_SC], inc[VR_SC];
#pragma unroll
        for (int j = 0; j < VR_SC; ++j) {
            const int p = c0 + 32 * j + lane;
            e[j] = (p < n) ? src[p] : 0.0;
            inc[j] = e[j];
        }
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
#pragma unroll
            for (int j = 0; j < VR_SC; ++j) {
                const double v = __shfl_up_sync(LTPL_FULL, inc[j], o);
                if (lane >= o) inc[j] += v;
            }
        }
        __syncwarp();   // every source element of the round is in a register: the in-place writes may start
#pragma unroll
        for (int j = 0; j < VR_SC; ++j) {
            const int p = c0 + 32 * j + lane;
            const double tot = __shfl_sync(LTPL_FULL, inc[j], 31);
            if (p < n) {
                const double sp = base + (inc[j] - e[j]);
                X0[p] = (float)(2.0 * e[j]);
                X4[p] = (float)sp;
                s_out[p] = sp;
            }
            base += tot;
        }
        __syncwarp();
    }
}

// STATE: stateful tick (ltpl_state.cuh) -- every path starts at its cut index + the vel_course rows (bf.trim), the planned
// velocity comes from bf.vel (= vel_plan in the library's launch), the follow-mode object distance from bf.obj_dist (k_ref)
// EXP1: friction-ellipse exponent 1.0 (LTPL:190 default): no pow on the chain
//
// Every device function with a long body has ONE call site (the sweeps are out of line on top): the rounds of the three
// warp roles (other class | follow warp 0 | follow warp 1) share one loop, so the kernel stays small in the instruction
// cache although six different profiles pass through it.
// GG: location dependent local_gg (buffers.gg, OTH:649-666): one more row per path (AX)
// No __grid_constant__ here: no parameter is copied to local memory, and with it the H100 timing is 2-4 % slower.
template <bool STATE, bool EXP1, bool GG>
__global__ void __launch_bounds__(VR_THREADS, 7)
k_vel_res(const LatDev lt, const LtplParams prm, const LtplDims dm, const LtplBuffers bf, const int nmax) {
    extern __shared__ __align__(16) unsigned char vr_smem[];
    __shared__ __align__(8) unsigned long long s_bar;
    __shared__ float s_tab[4 * VR_TAB];
    __shared__ int s_q[VR_P], s_n[VR_P], s_sh[VR_P], s_nb1[VR_P], s_nb2[VR_P], s_use_src[VR_P], s_row[VR_P], s_any_red;
    __shared__ long long s_in[VR_P], s_out[VR_P];
    __shared__ float s_wf0[VR_P], s_wcap[VR_P];
    __shared__ double s_v0[VR_P];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int B = dm.batch;
    const int nq = LTPL_NSLOT * B;
    const int nq_sub = LTPL_NSLOT * dm.sub_cnt;   // this launch's window: its own queues and fill counts
    const int* queue = bf.queue + 2 * LTPL_NSLOT * dm.sub_off;
    const int n_follow = bf.queue_cnt[4 + 4 * dm.sub_id], n_other = bf.queue_cnt[4 + 4 * dm.sub_id + 1];
    const int gf = (n_follow + VR_P - 1) / VR_P, go = (n_other + VR_P - 1) / VR_P;
    const int g = blockIdx.x;
    if (g >= gf + go) return;
    const bool follow_cls = g < gf;
    const size_t pplane = (size_t)nq * dm.p_max;
    const double* x_pl = bf.path;
    const double* y_pl = bf.path + pplane;
    const double* k_pl = bf.path + 3 * pplane;
    const double* e_pl = bf.path + 4 * pplane;
    double* s_pl = bf.s_vx_ax;
    double* vx_pl = s_pl + pplane;
    double* ax_pl = vx_pl + pplane;

    // ---- the group's paths ------------------------------------------------------------------------------------------
    if (tid == 0) s_any_red = 0;
    __syncthreads();
    if (tid < VR_P) {
        const int t = (follow_cls ? g : g - gf) * VR_P + tid;
        const bool live = t < (follow_cls ? n_follow : n_other);
        const int q = live ? queue[(follow_cls ? 0 : nq_sub) + t] : -1;
        int n = live ? bf.path_len[q] : 0;
        int off_in = 0, pref = 0;
        if (STATE && live) {
            pref = bf.trim[4 * q + 3];
            off_in = bf.trim[4 * q + 2] + pref;
            n = max(n - off_in, 0);
        }
        if (live && bf.vel[q % B] > prm.vel_max + 0.1) {   // VPFB:106 brake prefix: the reference raises (DESIGN.md 7)
            atomicOr(&bf.sc_flags[q % B], LTPL_SC_BRAKE_PREFIX);
            n = 0;
        }
        if (n > nmax) {   // cannot happen (nmax = dims.p_max); never write past the shared-memory rows
            atomicOr(&bf.sc_flags[q % B], LTPL_SC_CAPACITY);
            n = 0;
        }
        const long long ib = (long long)max(q, 0) * dm.p_max + off_in;
        s_q[tid] = (n > 0) ? q : -1;
        s_n[tid] = n;
        s_in[tid] = ib;
        s_out[tid] = (long long)max(q, 0) * dm.p_max + pref;
        s_sh[tid] = (int)(ib & 1);   // bulk copies start at an even element (16-byte source alignment)
        s_use_src[tid] = 0;
        s_row[tid] = -1;
        s_wf0[tid] = 0.0f;
        if (follow_cls && n > 0 && (bf.status[q] & LTPL_ST_REDUCED_HORIZON)) s_any_red = 1;
    }
    vr_stage_axm(prm, s_tab);
    if (tid == 0) vr_mbar_init(&s_bar, 1);
    __syncthreads();
    int np = 0;
#pragma unroll
    for (int r = 0; r < VR_P; ++r) np = max(np, s_n[r]);
    if (np == 0) return;
    const bool any_red = s_any_red != 0;

    // ---- one round of TMA bulk copies: el row -> X0 | X1, kappa row -> X2 | X3 of every path --------------------------
    const size_t rowf = (size_t)(GG ? 7 : 5) * nmax;   // floats per path block
    float* blk = reinterpret_cast<float*>(vr_smem);
    if (tid == 0) {
        unsigned total = 0;
        for (int r = 0; r < VR_P; ++r)
            if (s_n[r] > 0) total += 2u * 8u * (unsigned)((s_n[r] + s_sh[r] + 1) & ~1);
        vr_mbar_expect_tx(&s_bar, total);
        for (int r = 0; r < VR_P; ++r) {
            if (s_n[r] <= 0) continue;
            const unsigned bytes = 8u * (unsigned)((s_n[r] + s_sh[r] + 1) & ~1);
            float* X = blk + rowf * r;
            vr_bulk_g2s(X, e_pl + s_in[r] - s_sh[r], bytes, &s_bar);
            vr_bulk_g2s(X + 2 * (size_t)nmax, k_pl + s_in[r] - s_sh[r], bytes, &s_bar);
        }
    }
    const VRCfg c = vr_make_cfg(prm, s_tab);
    const float wmax = (float)(prm.vel_max * prm.vel_max);
    const double inv_ay = 1.0 / (prm.gg_ay * prm.gg_scale);
    const bool fw0 = follow_cls && warp == 0, fw1 = follow_cls && warp == 1;
    LTPL_PH_INIT

    // ---- follow, warp 1: opponent brake distance on the global race line, ggv = [100, 14, 14] (CVPF:134, 166-199);
    //      needs no path array and overlaps the bulk copies ----
    // the path a lane's chain works on: other class -> path 2 lane + warp (lanes < P / 2);  follow -> path lane (lanes < P;
    // warp 0: complete profile, warp 1: ego brake profile, then the control profile)
    const int pl = follow_cls ? lane % VR_P : min(2 * lane + warp, VR_P - 1);
    const bool lane_has = follow_cls ? (lane < VR_P) : (lane < VR_P / 2);
    const bool mine = lane_has && s_n[pl] > 0;
    const int q = s_q[pl], n = s_n[pl];
    const int b = mine ? q % B : 0;
    float* X = blk + rowf * pl;
    const float* E2 = X;
    float* WM = X + (size_t)nmax;
    const float* Kp = X + 2 * (size_t)nmax;
    float* SRC = X + 3 * (size_t)nmax;
    const float* S32 = X + 4 * (size_t)nmax;
    const float* AXp = X + 5 * (size_t)nmax;   // only with GG
    const float* IAYp = X + 6 * (size_t)nmax;  // only with GG
    const double* sg = s_pl + s_out[pl];
    const double vel_plan = mine ? bf.vel[b] : 0.0;
    const double vs_f = fmax(vel_plan, 0.0);
    const float wcap_m = (float)(vs_f * vs_f);
    if (mine) {   // first row: a profile that starts at the planned velocity returns it exactly (see the end)
        s_wcap[pl] = wcap_m;
        s_v0[pl] = vs_f;
    }
    int st = mine ? bf.status[q] : 0;
    const int action = mine ? bf.action_id[q] : LTPL_ACT_NONE;
    const bool red = (st & LTPL_ST_REDUCED_HORIZON) != 0;
    bool vel_bound = true;

    const int ng = lt.n_glob - 1;
    const double* __restrict__ G = lt.glob_rl;
    const double ov = (fw1 && mine) ? bf.cobj[4 * b + 2] : 0.0;
    const int start = (fw1 && mine) ? bf.cobj_start[b] : 0;
    double opp_stop_dist = 0.0;
    if (fw1 && mine) {
        const double dmq = prm.drag_coeff / prm.m_veh;
        double v0 = fmin(ov, G[6 * start + 4]);
        if (v0 < 0.0) v0 = 0.0;
        double ww = v0 * v0;
        int id = 0;
        while (id < ng && ww > 0.01) {   // four rows of the race line in flight per round trip
            double e4[4], k4[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                int r = start + id + u;
                while (r >= ng) r -= ng;
                e4[u] = G[6 * r + 5];
                k4[u] = fabs(G[6 * r + 3]);
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                if (id < ng && ww > 0.01) {
                    opp_stop_dist += e4[u];
                    ++id;
                    if (id <= ng - 1) {
                        const double a = acc_brake(ww, k4[u], 14.0, 1.0 / 14.0, prm.dyn_model_exp, dmq);
                        const double nx = fma(2.0 * a, e4[u], ww);
                        ww = (nx < 0.0) ? 0.0 : nx;
                    } else {
                        ww = 0.0;
                    }
                }
            }
        }
    }
    LTPL_PH(6)

    // ---- conversion of the staged rows.  other class: every warp its own paths; follow: warp 0 el (arc lengths, E2) of
    //      all paths, warp 1 kappa of all paths ----
    vr_mbar_wait(&s_bar, 0);
    LTPL_PH(0)
    for (int r = follow_cls ? 0 : warp; r < VR_P; r += (follow_cls ? 1 : 2)) {
        const int nr = s_n[r];
        if (nr <= 0) continue;
        float* Xr = blk + rowf * r;
        if (!fw0)
            vr_convert_kappa(Xr + 2 * (size_t)nmax, Xr + 5 * (size_t)nmax, Xr + 6 * (size_t)nmax, nr, s_sh[r], inv_ay,
                             GG ? bf.gg + s_in[r] : nullptr, pplane, prm.gg_scale, lane);
        if (!fw1) vr_convert_el(Xr, Xr + 4 * (size_t)nmax, s_pl + s_out[r], nr, s_sh[r], lane);
    }
    LTPL_PH(1)
    if (fw1) {
        vr_bar_arrive(1);
        // ---- nearest path point to the object and to the ego position (OTH:774-782), first ticks only: 32 / VR_P lanes
        //      per path, all paths of the group at once (the loads of one lane are independent) ----
        if (!STATE) {
            constexpr int LPP = 32 / VR_P;
            const int r = lane / LPP, sub = lane % LPP;
            const int nr = s_n[r];
            const int br = (nr > 0) ? s_q[r] % B : 0;
            const double ox = bf.cobj[4 * br], oy = bf.cobj[4 * br + 1];
            const double epx = bf.pos[2 * br], epy = bf.pos[2 * br + 1];
            const double* xr = x_pl + s_in[r];
            const double* yr = y_pl + s_in[r];
            double bv1 = LTPL_INF, bv2 = LTPL_INF;
            int i1 = 0x7fffffff, i2 = 0x7fffffff;
#pragma unroll 1
            for (int p0 = sub; p0 < nr; p0 += 8 * LPP) {   // 16 loads of a lane in flight; points visited in index order
                double xx[8], yy[8];
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                    const int p = min(p0 + u * LPP, nr - 1);
                    xx[u] = xr[p];
                    yy[u] = yr[p];
                }
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                    const int p = p0 + u * LPP;
                    const double d1 = dist2_rn(xx[u], yy[u], ox, oy), d2 = dist2_rn(xx[u], yy[u], epx, epy);
                    if (p < nr && d1 < bv1) {
                        bv1 = d1;
                        i1 = p;
                    }
                    if (p < nr && d2 < bv2) {
                        bv2 = d2;
                        i2 = p;
                    }
                }
            }
#pragma unroll
            for (int o = 1; o < LPP; o <<= 1) {   // first minimum within the lane group: (value, index) lexicographic
                const double u1 = __shfl_xor_sync(LTPL_FULL, bv1, o), u2 = __shfl_xor_sync(LTPL_FULL, bv2, o);
                const int j1 = __shfl_xor_sync(LTPL_FULL, i1, o), j2 = __shfl_xor_sync(LTPL_FULL, i2, o);
                if (u1 < bv1 || (u1 == bv1 && j1 < i1)) {
                    bv1 = u1;
                    i1 = j1;
                }
                if (u2 < bv2 || (u2 == bv2 && j2 < i2)) {
                    bv2 = u2;
                    i2 = j2;
                }
            }
            if (sub == 0 && nr > 0) {
                s_nb1[r] = i1;
                s_nb2[r] = i2;
            }
            __syncwarp();
        }
        LTPL_PH(8)
    } else if (fw0) {
        vr_bar_arrive(2);   // E2 and the arc lengths are ready for warp 1
        vr_bar_sync(1);     // K' of warp 1 has landed
    } else {
        __threadfence_block();
        __syncwarp();
    }

    // ==================================================================================================================
    // rounds of (forward sweep, backward sweep):
    //   other class        round 0: v_end rule + one profile (OTH:834-923)
    //   follow, warp 0     round 0: complete profile (CVPF:296);  round 2 (a reduced-horizon path in the group): second
    //                      profile with v_end = 0 (OTH:846-923)
    //   follow, warp 1     round 0: ego brake profile (CVPF:152-165, forward only, float64 accumulator);  round 1: follow
    //                      scalars (CVPF:139-247), then the control profile -- both warps' chains advance concurrently
    // ==================================================================================================================
    int flags = 0, idx_c = 0, stop_idx = 0, hi = -1;
    bool use_prof = false, has_ctrl = false;
    double vcs = 0.0;
    const int rounds = follow_cls ? (any_red ? 3 : 2) : 1;
#pragma unroll 1
    for (int round = 0; round < rounds; ++round) {
        bool on = false;
        int lo = 0;
        float wcap = wcap_m, we = -1.0f, wmx = wmax;
        float* W = WM;
        bool brake = false;
        hi = -1;
        if (round == 2) {   // materialise min(profile, complete) first: quirk q1 compares it with the second profile
            for (int r = 0; r < VR_P; ++r) {
                float* Wr = blk + rowf * r + nmax;
                const float* Sr = blk + rowf * r + 3 * (size_t)nmax;
                for (int p = tid; p < s_n[r]; p += VR_THREADS) Wr[p] = fminf(Sr[p], Wr[p]);
            }
            __syncthreads();
        }
        if (!follow_cls || (fw0 && round == 2)) {
            // ---- single profile: all actions but follow, and follow with a reduced horizon ----
            on = mine && (!follow_cls || red);
            if (on) {
                double v_end;
                int v_idx;
                if (red) {
                    v_end = 0.0;
                    // first i with cumsum(el[:-1])[i] >= spl_len - 5  <=>  s[i + 1] >= spl_len - 5   (OTH:851-859)
                    const double spl_len = __ldcg(sg + n - 1);
                    int first = vr_first_ge_s(S32 + 1, sg + 1, n - 1, spl_len - 5.0);
                    if (first >= n - 1) first = 0;
                    v_idx = first + 1;
                    if (v_idx == 1 && n > 1) v_idx = n;
                } else {
                    const int nn = bf.n_nodes[q];
                    const int* nd = bf.nodes + ((size_t)q * dm.h_max + (nn - 1)) * 2;
                    const int end_layer = nd[0], end_node = nd[1];
                    int dn = end_node - lt.rl_idx[end_layer];
                    if (dn < 0) dn = -dn;
                    const double raceline_offset = dn * lt.lat_offset;   // quirk q3
                    v_end = lt.vel_rl[end_layer];
                    v_end -= fmin(v_end * lt.vel_decrease_lat * raceline_offset, v_end);
                    v_idx = n;
                }
                if (v_idx > 1) {
                    hi = v_idx - 1;
                    const double ve = fmax(v_end, 0.0);
                    we = (float)(ve * ve);
                }
                if (follow_cls) W = SRC;   // second profile of a follow path: SRC is free after the merge above
            }
        } else if (fw0 && round == 0) {
            // ---- complete profile on [0, n-1] (CVPF:296) ----
            on = mine;
            hi = n - 1;
        } else if (fw1 && round == 0) {
            // ---- ego brake profile on [0, n-1] into SRC (CVPF:152-165) ----
            LTPL_PH(7)
            vr_bar_sync(2);   // E2 and the arc lengths of warp 0 are ready
            LTPL_PH(9)
            on = mine;
            brake = true;
            hi = n - 1;
            W = SRC;
        } else if (fw1 && round == 1) {
            // ---- follow scalars (CVPF:139-247), then the control profile on [idx_c, stop_idx] into SRC ----
            double v_end_c = 0.0, v_control = 0.0;
            if (mine) {
                double obj_dist;
                if (STATE) {
                    obj_dist = bf.obj_dist[b];
                } else {
                    const double* xr = x_pl + s_in[pl];
                    const double* yr = y_pl + s_in[pl];
                    const double* er = e_pl + s_in[pl];
                    const double s_obj = vr_s_coord_from_nb(xr, yr, er, sg, n, s_nb1[pl], bf.cobj[4 * b], bf.cobj[4 * b + 1]);
                    const double s_start = vr_s_coord_from_nb(xr, yr, er, sg, n, s_nb2[pl], bf.pos[2 * b], bf.pos[2 * b + 1]);
                    obj_dist = s_obj - s_start;   // OTH:784
                }
                const double v_ego = bf.vel_est[b];
                const double control_d = prm.follow_c_p * prm.safety_d + lt.veh_length;
                const double safety_d = prm.safety_d + lt.veh_length;
                if ((obj_dist - safety_d) < 0) flags |= 1;
                // ego stop distance: summed el while the brake profile is above 0.1 m/s (CVPF:161-165)
                const int pz = vr_first_le(SRC, n, 0.01f);
                const double ego_stop_dist = (pz < n) ? __ldcg(sg + pz) : __ldcg(sg + n - 1) + (e_pl + s_in[pl])[n - 1];
                const double s_stop = obj_dist - safety_d + opp_stop_dist;   // CVPF:201-223
                stop_idx = min(vr_first_ge_s(S32, sg, n, s_stop), n - 1);
                const double s_last = __ldcg(sg + n - 1);
                if (s_stop > s_last) {
                    const double s_ends = opp_stop_dist - (s_stop - s_last);
                    int idx = 0;
                    double s_summed = 0.0;
                    while (s_summed < s_ends && idx < ng) {   // four rows in flight per round trip
                        double e4[4];
#pragma unroll
                        for (int u = 0; u < 4; ++u) {
                            int r4 = start + idx + u;
                            while (r4 >= ng) r4 -= ng;
                            e4[u] = G[6 * r4 + 5];
                        }
#pragma unroll
                        for (int u = 0; u < 4; ++u)
                            if (s_summed < s_ends && idx < ng) {
                                s_summed += e4[u];
                                ++idx;
                            }
                    }
                    int r = start + idx;
                    while (r >= ng) r -= ng;
                    v_end_c = G[6 * r + 4];
                }
                if (prm.follow_control_type == 0) {   // CVPF:28-75
                    v_control = ov - prm.follow_k_p * (control_d - obj_dist) + prm.follow_k_d * (ov - v_ego);
                } else {
                    double arg = (control_d - obj_dist) * LTPL_PI / 2 * 1 / prm.follow_tan_w;
                    arg = fmin(fmax(arg, -LTPL_PI / 2 + 1e-5), LTPL_PI / 2 - 1e-5);
                    v_control = ov - tan(arg) * prm.follow_k_p + prm.follow_k_d * (ov - v_ego);
                }
                v_control = fmin(fmax(v_control, 0.0), prm.vel_max);
                if (ego_stop_dist < s_stop) {   // CVPF:247-292
                    use_prof = true;
                    if (vel_plan > v_control && stop_idx >= 2) {
                        int first = vr_first_le(SRC, n, (float)(v_control * v_control));
                        if (first >= n) first = 0;   // np.argmax of an all-False array
                        idx_c = min(first, stop_idx);
                        if (idx_c == 0) idx_c = stop_idx;
                        vcs = sqrt((double)SRC[idx_c]);
                    } else {
                        if (!(stop_idx >= 2)) flags |= 2;
                        idx_c = 0;
                        vcs = vel_plan;
                    }
                    has_ctrl = (stop_idx - idx_c) > 0;
                }
            }
            const double vcs_p = fmax(vcs, 0.0), vec_p = fmax(v_end_c, 0.0);
            on = mine && use_prof && has_ctrl;
            lo = idx_c;
            hi = on ? stop_idx : -1;
            wcap = (float)(vcs_p * vcs_p);
            we = (float)(vec_p * vec_p);
            wmx = (float)(v_control * v_control);
            W = SRC;
            LTPL_PH(10)
        }

        if (fw1 && round == 0) {
            vr_brake<EXP1, GG>(c, on, Kp, E2, AXp, W, lo, hi, wcap, we, nmax);
        } else {
            vr_forward<EXP1, GG>(c, on, Kp, E2, AXp, W, lo, hi, wcap, we, wmx, nmax);
            if (fw0 && round == 0) {
                LTPL_PH(3)
            }
        }
        const float w_first = vr_backward<EXP1, GG>(c, on && !brake, Kp, E2, AXp, IAYp, W, lo, hi, wmx);

        if (!follow_cls || (fw0 && round == 2)) {
            if (on) {
                for (int p = hi + 1; p < n; ++p) W[p] = 0.0f;   // zeros behind the reduced horizon (OTH:900-903)
                const float wf0 = (hi >= 0) ? w_first : 0.0f;
                if (follow_cls) {
                    s_wf0[pl] = wf0;
                    s_use_src[pl] = (n >= 6 && !(WM[5] < SRC[5])) ? 1 : 0;   // quirk q1 (OTH:923): row 5 decides
                } else {
                    vel_bound = fabs(sqrt((double)wf0) - vel_plan) < prm.v_max_offset;
                }
            }
        } else if (fw1 && round == 1) {
            if (mine && use_prof) {
                const double vcs_p = fmax(vcs, 0.0);
                if (!has_ctrl) SRC[idx_c] = (float)(vcs_p * vcs_p);
                for (int p = stop_idx + 1; p < n; ++p) SRC[p] = 0.0f;
                const double v0c = has_ctrl ? sqrt((double)w_first) : vcs;
                if (has_ctrl && fabs(v0c - vcs) > 1.0) flags |= 2;
                const double prof0 = (idx_c == 0) ? v0c : vs_f;
                if (fabs(prof0 - vel_plan) > 1.0) flags |= 2;
            }
            if (flags & 1) st |= LTPL_ST_TOO_CLOSE;
            vel_bound = !(flags & 2);
            LTPL_PH(11)
        } else if (fw0 && round == 0) {
            LTPL_PH(4)
        }
        if (follow_cls && round >= 1)   // (round 0 -> 1: warp 1 only depends on its own brake profile)
            __syncthreads();
        else
            __syncwarp();
        if (follow_cls && round == 1) {
            LTPL_PH(5 + 7 * warp)
        }
    }

    // ---- acceptance (OTH:943-1025; no backup plan exists on the first tick); the compact export row of a kept trajectory
    //      is taken here so that the element-wise end can write it ----
    if (mine && !fw0) {
        if (follow_cls && red) vel_bound = fabs(sqrt((double)s_wf0[pl]) - vel_plan) < prm.v_max_offset;
        if (!vel_bound) st |= LTPL_ST_VEL_BOUND_VIOL;
        // stateful tick: a backup plan exists (OTH:325-344), so a straight / follow profile that breaks the bound is
        // replaced by a brake profile on the OLD path (OTH:950-1006): flag here, k_backup plans it and clears the flag (no
        // backup plan exists after an invalid last solution, const_len == 0, or a restart, st_info[0] < 0: the profile is
        // kept, OTH:945-948)
        if (STATE && !vel_bound && (action == LTPL_ACT_FOLLOW || action == LTPL_ACT_STRAIGHT) && bf.const_len[b] != 0 &&
            bf.st_info[8 * (size_t)b] >= 0)
            atomicOr(&bf.sc_flags[b], LTPL_SC_STATE_FALLBACK | (6 << LTPL_SC_REASON_SHIFT));
        if (vel_bound || action == LTPL_ACT_FOLLOW || action == LTPL_ACT_STRAIGHT) {
            st |= LTPL_ST_TRAJ_VALID;
            bf.traj_len[q] = min(n, dm.n_export);
            bf.traj_id[q] = prm.traj_base_id + action;
            const int e = atomicAdd(&bf.queue_cnt[2], 1);
            bf.exp_q[e] = q;
            bf.traj_row[q] = e;
            s_row[pl] = e;
        }
        bf.status[q] = st;
    }
    if (follow_cls)
        __syncthreads();
    else
        __syncwarp();

    // ---- element-wise end: min(src, complete) (CVPF:297-310), vx = sqrt(w), ax = (w1 - w0) / (2 ds), standstill fix-up
    //      (OTH:926-941); follow: all 64 threads over all paths, other class: every warp over its own paths.
    //      First ticks also write the exported rows (s, x, y, psi, kappa, vx, ax as fp32, cut to nmbr_export_points:
    //      OTH:941 + LTPL:401-406) of the kept trajectories here -- no separate export kernel, s / vx / ax go out from
    //      shared memory; stateful ticks export behind k_prefix (vel_course rows in front, ltpl_state.cuh) ----
    {
        const int t0 = follow_cls ? tid : lane, tstep = follow_cls ? VR_THREADS : 32;
        for (int r = follow_cls ? 0 : warp; r < VR_P; r += (follow_cls ? 1 : 2)) {
            const int nr = s_n[r];
            if (nr <= 0) continue;
            const float* Er = blk + rowf * r;
            const float* Wr = Er + nmax;
            const float* Sr = Er + 3 * (size_t)nmax;
            const float* S32r = Er + 4 * (size_t)nmax;
            // 0: min(SRC, W) (follow), 1: W (other class; follow after the merge of round 1), 2: SRC (q1 took the second)
            const int mode = !follow_cls ? 1 : (any_red ? (s_use_src[r] ? 2 : 1) : 0);
            for (int p = t0; p < nr; p += tstep) {
                const float w0 = (mode == 0) ? fminf(Sr[p], Wr[p]) : ((mode == 1) ? Wr[p] : Sr[p]);
                float a = 0.0f;
                if (p < nr - 1) {
                    const float w1 = (mode == 0) ? fminf(Sr[p + 1], Wr[p + 1]) : ((mode == 1) ? Wr[p + 1] : Sr[p + 1]);
                    a = (w1 - w0) * vr_rcp(Er[p]);
                    if (w0 <= 1e-16f && fabsf(a) <= 1e-8f) a = -5.0f;
                }
                // v[0] = min(v[0], v_start) (tph): an unchanged first value IS the planned velocity, bit for bit
                const double v = (p == 0 && w0 == s_wcap[r]) ? s_v0[r] : (double)sqrtf(w0);
                vx_pl[s_out[r] + p] = v;
                ax_pl[s_out[r] + p] = (double)a;
            }
            // exported rows: four points of a thread in flight (16 independent loads), then their 28 stores
            const int er = STATE ? -1 : s_row[r];
            const int ne = (er >= 0) ? min(nr, dm.n_export) : 0;
            float* __restrict__ out = bf.traj + (size_t)max(er, 0) * dm.n_export * 7;
            const double* __restrict__ ppr = bf.path + s_in[r];
#pragma unroll 1
            for (int p0 = t0; p0 < ne; p0 += 4 * tstep) {
                double g[4][4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int p = min(p0 + u * tstep, ne - 1);
#pragma unroll
                    for (int cc = 0; cc < 4; ++cc) g[u][cc] = ppr[cc * pplane + p];
                }
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int p = p0 + u * tstep;
                    if (p < ne) {
                        const float w0 = (mode == 0) ? fminf(Sr[p], Wr[p]) : ((mode == 1) ? Wr[p] : Sr[p]);
                        float a = 0.0f;
                        if (p < nr - 1) {
                            const float w1 = (mode == 0) ? fminf(Sr[p + 1], Wr[p + 1])
                                                         : ((mode == 1) ? Wr[p + 1] : Sr[p + 1]);
                            a = (w1 - w0) * vr_rcp(Er[p]);
                            if (w0 <= 1e-16f && fabsf(a) <= 1e-8f) a = -5.0f;
                        }
                        float* o = out + (size_t)p * 7;
                        o[0] = S32r[p];
                        o[1] = (float)g[u][0];
                        o[2] = (float)g[u][1];
                        o[3] = (float)g[u][2];
                        o[4] = (float)g[u][3];
                        o[5] = (p == 0 && w0 == s_wcap[r]) ? (float)s_v0[r] : sqrtf(w0);
                        o[6] = a;
                    }
                }
            }
        }
    }
    LTPL_PH(13)
}
