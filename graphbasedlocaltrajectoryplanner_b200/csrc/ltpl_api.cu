// ltpl_api.cu -- C-ABI of libltpl_b200.so (include/ltpl_b200.h).  Host side only resolves pointers and launches
// kernels on the caller's stream; no allocation, no synchronisation on the hot path.
//
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -fmad=false -shared -Xcompiler -fPIC
#include <atomic>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <new>
#include <string>

#include "ltpl_path.cuh"
#include "ltpl_plan.cuh"
#include "ltpl_vel.cuh"
#include "ltpl_vel_res.cuh"
#include "ltpl_velprofile.cuh"
#include "ltpl_emerg.cuh"
#include "ltpl_state.cuh"
#include "ltpl_smooth.cuh"

static std::atomic<unsigned long long> g_launches{0};

static thread_local std::string g_err;

static int fail(const char* what) {
    g_err = what;
    return -1;
}

static int check_launch(const char* name) {
    g_launches.fetch_add(1, std::memory_order_relaxed);
    cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) {
        g_err = std::string(name) + ": " + cudaGetErrorString(e);
        (void)cudaGetLastError();
        return -2;
    }
    return 0;
}

// CTAs of a launch with one warp per scenario / path
static int ctas(int warps, int warps_per_cta = LTPL_WARPS_PER_CTA) { return (warps + warps_per_cta - 1) / warps_per_cta; }
static const int kThreads = LTPL_WARPS_PER_CTA * 32;

// Dynamic shared memory of a kernel family: a size above the 200 KB cap is refused, a size above the 48 KB default is
// allowed by cudaFuncSetAttribute on every kernel of the family.  The attribute belongs to the kernel on the current
// device and is shared by every handle and thread there, so it is only ever raised (another handle may rely on a larger
// value), under a lock.  The size a handle has made sure of is kept per handle (one handle, one device) to skip the calls.
enum SmemFamily { kSmemFollow, kSmemPlan, kSmemPath, kSmemVel };
static const size_t kSmemCap = 200 * 1024;
static std::mutex g_smem_lock;

template <class Fn, size_t N>
static int allow_smem(const LtplLattice* lat, SmemFamily fam, size_t smem, Fn const (&fns)[N], const char* name,
                      const char* too_large) {
    if (smem > kSmemCap) return fail(too_large);
    if (smem > 48 * 1024 && smem > lat->smem_allowed[fam]) {
        std::lock_guard<std::mutex> lock(g_smem_lock);
        for (Fn f : fns) {
            cudaFuncAttributes a;
            cudaError_t e = cudaFuncGetAttributes(&a, (const void*)f);
            if (e == cudaSuccess && (size_t)a.maxDynamicSharedSizeBytes < smem)
                e = cudaFuncSetAttribute((const void*)f, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (e != cudaSuccess) {
                (void)cudaGetLastError();
                g_err = std::string(name) + ": dynamic shared-memory attribute: " + cudaGetErrorString(e);
                return -2;
            }
        }
        lat->smem_allowed[fam] = smem;
    }
    return 0;
}

// k_plan's per-warp shared memory: node rows of maxn entries, bits of the edge window
static int plan_maxn(const LtplLatticeHeader* h) { return ((h->max_nodes_per_layer + 31) / 32) * 32; }
static int plan_mask_words(const LtplLatticeHeader* h) { return (h->max_window_edges + 31) / 32 + 1; }

// largest dims.k_obj whose k_plan shared memory stays within kSmemCap; 0: not even the lattice window fits
static int max_objects(const LtplLatticeHeader* h, int h_max) {
    const int maxn = plan_maxn(h), mw = plan_mask_words(h);
    const size_t per_warp = kSmemCap / LTPL_WARPS_PER_CTA;
    const size_t base = plan_smem_bytes_per_warp(maxn, h_max, mw, 0);
    if (base > per_warp) return 0;
    int k = (int)((per_warp - base) / sizeof(VehRec));
    while (k > 0 && plan_smem_bytes_per_warp(maxn, h_max, mw, k) > per_warp) --k;
    return k;
}

// k_plan<ZONE, STATE, DENSE>: one warp per scenario (ltpl_plan.cuh), [ZONE + 2 STATE + 4 DENSE]
typedef void (*PlanFn)(const __grid_constant__ LatDev, const __grid_constant__ LtplParams, const __grid_constant__ LtplDims,
                       const __grid_constant__ LtplBuffers, const int, const int, const int);
static const PlanFn kPlanFns[8] = {k_plan<false, false, false>, k_plan<true, false, false>, k_plan<false, true, false>,
                                   k_plan<true, true, false>,   k_plan<false, false, true>, k_plan<true, false, true>,
                                   k_plan<false, true, true>,   k_plan<true, true, true>};

static int launch_k_plan(const LtplLattice* lat, const LtplParams* prm, const LtplDims* dm, const LtplBuffers* bf,
                         cudaStream_t st, bool stateful) {
    const int maxn = plan_maxn(&lat->h);
    const int hl = dm->h_max;
    const int mask_words = plan_mask_words(&lat->h);
    const size_t smem = plan_smem_bytes_per_warp(maxn, hl, mask_words, dm->k_obj) * LTPL_WARPS_PER_CTA;
    if (int r = allow_smem(lat, kSmemPlan, smem, kPlanFns, "k_plan", "lattice window too large for shared memory"))
        return r;
    // Shared-memory carveout: what LTPL_PLAN_MINB CTAs need with at least 16 object slots (1 KB reserved per CTA, 228 KB
    // per sm_90 SM).  For fewer slots the driver would pick a smaller carveout (more L1) for k_plan, and the benchmark
    // then runs about 4 % slower on an H100: k_vel_res of the other scenario windows, which needs the largest carveout,
    // slows down beside it (DESIGN.md section 5).  The attribute is a hint shared by every handle on the device.
    const size_t need = (plan_smem_bytes_per_warp(maxn, hl, mask_words, dm->k_obj < 16 ? 16 : dm->k_obj) *
                         LTPL_WARPS_PER_CTA + 1024) * LTPL_PLAN_MINB;
    const int carveout = (int)((need * 100 + 228 * 1024 - 1) / (228 * 1024));
    if (carveout != lat->plan_carveout) {
        for (PlanFn f : kPlanFns)
            if (cudaFuncSetAttribute((const void*)f, cudaFuncAttributePreferredSharedMemoryCarveout,
                                     carveout < 100 ? carveout : 100) != cudaSuccess) {
                (void)cudaGetLastError();
                return fail("k_plan: shared-memory carveout attribute");
            }
        lat->plan_carveout = carveout;
    }
    const bool zone = dm->n_zones > 0;
    const bool dense = lat->h.num_edges >= 2 * lat->h.num_nodes;   // in-edges per node (dp_run<.., DENSE>)
    kPlanFns[(zone ? 1 : 0) + (stateful ? 2 : 0) + (dense ? 4 : 0)]<<<ctas(dm->sub_cnt), kThreads, smem, st>>>(
        lat->d, *prm, *dm, *bf, maxn, hl, mask_words);
    return check_launch("k_plan");
}

// k_path<STATE>: one warp per path (ltpl_path.cuh)
static int launch_k_path(const LtplLattice* lat, const LtplParams* prm, const LtplDims* dm, const LtplBuffers* bf,
                         cudaStream_t st, bool stateful) {
    const size_t smem = path_smem_bytes_per_warp(dm->h_max) * LTPL_WARPS_PER_CTA;
    typedef void (*PathFn)(const __grid_constant__ LatDev, const __grid_constant__ LtplParams,
                           const __grid_constant__ LtplDims, const __grid_constant__ LtplBuffers);
    static const PathFn fns[2] = {k_path<false>, k_path<true>};
    if (int r = allow_smem(lat, kSmemPath, smem, fns, "k_path", "lattice window too large for shared memory")) return r;
    fns[stateful]<<<ctas(LTPL_NSLOT * dm->sub_cnt), kThreads, smem, st>>>(lat->d, *prm, *dm, *bf);
    return check_launch("k_path");
}

// velocity kernel: one CTA per VR_P queued paths of one class, the paths resident in shared memory (ltpl_vel_res.cuh)
static int launch_k_vel(const LtplLattice* lat, const LtplParams* prm, const LtplDims* dm, const LtplBuffers* bf,
                        cudaStream_t st, bool stateful) {
    const int nmax = dm->p_max;
    if (nmax > 32 * VR_MAXM)
        return fail("k_vel: dims.p_max exceeds the shared-memory capacity of the velocity kernel (<= 512)");
    const bool gg = bf->gg != nullptr;   // location dependent local_gg: the general-exponent variant carries it
    const size_t smem = vr_smem_bytes(nmax, gg);
    typedef void (*VelFn)(const LatDev, const LtplParams, const LtplDims, const LtplBuffers, const int);
    // <STATE, EXP1, GG>: [stateful + 2 * (0 exponent 1, 1 general exponent, 2 local_gg planes)]
    static const VelFn fns[6] = {k_vel_res<false, true, false>, k_vel_res<true, true, false>,
                                 k_vel_res<false, false, false>, k_vel_res<true, false, false>,
                                 k_vel_res<false, false, true>, k_vel_res<true, false, true>};
    if (int r = allow_smem(lat, kSmemVel, smem, fns, "k_vel", "dims.p_max too large for the velocity kernel's shared memory"))
        return r;
    const int kind = gg ? 2 : (prm->dyn_model_exp == 1.0 ? 0 : 1);
    const int nq = LTPL_NSLOT * dm->sub_cnt;   // paths of this launch's scenario window
    const int grid = nq / VR_P + 2;            // >= groups of the follow queue + groups of the other queue
    fns[(stateful ? 1 : 0) + 2 * kind]<<<grid, VR_THREADS, smem, st>>>(lat->d, *prm, *dm, *bf, nmax);
    return check_launch("k_vel");
}

extern "C" {

int ltpl_version(void) { return LTPL_ABI_VERSION; }

const char* ltpl_last_error(void) { return g_err.c_str(); }

uint64_t ltpl_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

int ltpl_sizeof(int which) {
    switch (which) {
        case 0: return (int)sizeof(LtplLatticeHeader);
        case 1: return (int)sizeof(LtplParams);
        case 2: return (int)sizeof(LtplDims);
        case 3: return (int)sizeof(LtplBuffers);
        case 4: return (int)sizeof(LtplVelBatch);
        default: return -1;
    }
}

int ltpl_max_objects(const LtplLatticeHeader* h, int h_max) { return h ? max_objects(h, h_max) : -1; }

int ltpl_lattice_create(const LtplLatticeHeader* h, void* dev_blob, LtplLattice** out) {
    if (!h || !dev_blob || !out) return fail("ltpl_lattice_create: null argument");
    if (h->abi_version != LTPL_ABI_VERSION) return fail("ltpl_lattice_create: ABI version mismatch");
    if (h->max_nodes_per_layer > 64 || h->max_nodes_per_layer < 1)
        return fail("ltpl_lattice_create: max_nodes_per_layer must be in [1, 64]");
    if (h->tab_stride < 3 || h->tab_stride > 255) return fail("ltpl_lattice_create: tab_stride must be in [3, 255]");
    if (h->num_layers < 4) return fail("ltpl_lattice_create: lattice needs at least 4 layers");
    if (h->grid_nx < 1 || h->grid_ny < 1 || !(h->grid_inv_cell > 0.0)) return fail("ltpl_lattice_create: nearest-vertex grid missing");
    LtplLattice* lat = new (std::nothrow) LtplLattice;
    if (!lat) return fail("ltpl_lattice_create: out of host memory");
    lat->h = *h;
    unsigned char* p = static_cast<unsigned char*>(dev_blob);
    LatDev& d = lat->d;
    d.L = h->num_layers;
    d.Nn = h->num_nodes;
    d.E = h->num_edges;
    d.S = h->num_samples;
    d.n_glob = h->n_glob_rl;
    d.closed = h->closed;
    d.plan_mode = h->plan_horizon_mode;
    d.max_nodes = h->max_nodes_per_layer;
    d.max_window_edges = h->max_window_edges;
    d.lat_offset = h->lat_offset;
    d.lat_res = h->lat_resolution;
    d.step = h->sampled_resolution;
    d.vel_decrease_lat = h->vel_decrease_lat;
    d.veh_width = h->veh_width;
    d.veh_length = h->veh_length;
    d.virt_cost = h->virt_goal_node_cost;
    d.min_plan_horizon = h->min_plan_horizon;
#define LTPL_PTR(field, type, off) d.field = reinterpret_cast<const type*>(p + h->off)
    LTPL_PTR(node_off, int, off_node_off);
    LTPL_PTR(rl_idx, int, off_raceline_index);
    LTPL_PTR(s_rl, double, off_s_raceline);
    LTPL_PTR(vel_rl, double, off_vel_raceline);
    LTPL_PTR(refline, double2, off_refline);
    LTPL_PTR(raceline, double2, off_raceline);
    LTPL_PTR(bound1, double2, off_bound1);
    LTPL_PTR(bound2, double2, off_bound2);
    LTPL_PTR(center, double2, off_centerline);
    LTPL_PTR(node_xy, double2, off_node_xy);
    LTPL_PTR(node_psi, double, off_node_psi);
    LTPL_PTR(node_layer, int, off_node_layer);
    LTPL_PTR(in_off, int2, off_in_off);
    LTPL_PTR(edge_layer_off, int, off_edge_layer_off);
    LTPL_PTR(edge_src, int, off_edge_src);
    LTPL_PTR(edge_dst, int, off_edge_dst);
    LTPL_PTR(edge_cost, double, off_edge_cost);
    LTPL_PTR(edge_len, double, off_edge_len);
    LTPL_PTR(edge_psi1, double, off_edge_psi1);
    LTPL_PTR(edge_psi0, double, off_edge_psi0);
    LTPL_PTR(samp_off, int, off_samp_off);
    LTPL_PTR(samp_xy, double2, off_samp_xy);
    LTPL_PTR(samp_el, double, off_samp_el);
    LTPL_PTR(samp_edge, int, off_samp_edge);
    LTPL_PTR(glob_rl, double, off_glob_rl);
    LTPL_PTR(glob_xy, double2, off_glob_xy);
    LTPL_PTR(edge_rec, LtplEdgeRec, off_edge_rec);
    LTPL_PTR(tab_reach, int, off_tab_reach);
    LTPL_PTR(tab_node, unsigned char, off_tab_node);
    LTPL_PTR(tab_edge, int, off_tab_edge);
    LTPL_PTR(grid_center, int, off_grid_center);
    LTPL_PTR(grid_refline, int, off_grid_refline);
    LTPL_PTR(grid_raceline, int, off_grid_raceline);
    LTPL_PTR(grid_glob, int, off_grid_glob);
#undef LTPL_PTR
    d.grid_nx = h->grid_nx;
    d.grid_ny = h->grid_ny;
    d.grid_cyclic = h->closed;
    d.grid_x0 = h->grid_x0;
    d.grid_y0 = h->grid_y0;
    d.grid_inv_cell = h->grid_inv_cell;
    d.tab_stride = h->tab_stride;
    {  // follow table: one warp per node (k_follow_table), once per lattice
        const int maxn = ((h->max_nodes_per_layer + 31) / 32) * 32;
        const size_t smem = table_smem_bytes_per_warp(maxn, h->tab_stride) * LTPL_WARPS_PER_CTA;
        if (int r = allow_smem(lat, kSmemFollow, smem, {k_follow_table}, "k_follow_table",
                               "ltpl_lattice_create: planning range too large for shared memory")) {
            delete lat;
            return r;
        }
        k_follow_table<<<ctas(h->num_nodes), kThreads, smem>>>(d, maxn, reinterpret_cast<int*>(p + h->off_tab_reach),
                                                              p + h->off_tab_node, reinterpret_cast<int*>(p + h->off_tab_edge));
        cudaError_t e = cudaGetLastError();
        if (e == cudaSuccess) e = cudaDeviceSynchronize();
        if (e != cudaSuccess) {
            g_err = std::string("ltpl_lattice_create: k_follow_table: ") + cudaGetErrorString(e);
            delete lat;
            return -2;
        }
        g_launches.fetch_add(1, std::memory_order_relaxed);
    }
    {   // internal streams / events of the scenario windows (ltpl_set_subbatches)
        cudaError_t e = cudaEventCreateWithFlags(&lat->ev_fork, cudaEventDisableTiming);
        for (int i = 0; i < LTPL_MAX_SUB - 1 && e == cudaSuccess; ++i) {
            e = cudaStreamCreateWithFlags(&lat->aux[i], cudaStreamNonBlocking);
            if (e == cudaSuccess) e = cudaEventCreateWithFlags(&lat->ev_join[i], cudaEventDisableTiming);
        }
        if (e != cudaSuccess) {
            g_err = std::string("ltpl_lattice_create: streams: ") + cudaGetErrorString(e);
            ltpl_lattice_destroy(lat);
            return -2;
        }
        lat->n_sub = LTPL_DEFAULT_SUB;
        lat->sub_min = LTPL_SUB_MIN;
        if (const char* env = getenv("LTPL_SUBBATCHES")) {
            const int n = atoi(env);
            if (n >= 1 && n <= LTPL_MAX_SUB) lat->n_sub = n;
        }
    }
    *out = lat;
    return 0;
}

int ltpl_lattice_destroy(LtplLattice* lat) {
    if (!lat) return 0;
    for (int i = 0; i < LTPL_MAX_SUB - 1; ++i) {
        if (lat->aux[i]) cudaStreamDestroy(lat->aux[i]);
        if (lat->ev_join[i]) cudaEventDestroy(lat->ev_join[i]);
    }
    if (lat->ev_fork) cudaEventDestroy(lat->ev_fork);
    delete lat;
    return 0;
}

int ltpl_set_subbatches(LtplLattice* lat, int n) {
    if (!lat) return fail("null argument");
    if (n < 1 || n > LTPL_MAX_SUB) return fail("ltpl_set_subbatches: n must be in [1, LTPL_MAX_SUB]");
    lat->n_sub = n;
    lat->sub_min = 1;   // an explicit request is taken literally (windows of at least one scenario)
    return 0;
}

// ---- scenario windows: the launches of one call run per window, window 0 on the caller's stream, the others on the
// handle's internal streams between an event fork and an event join (also valid under stream capture) ----
static LtplDims window_dims(const LtplDims* dm, int s, int n) {
    LtplDims w = *dm;
    const int per = (dm->batch + n - 1) / n;
    w.sub_id = s;
    w.sub_off = s * per;
    w.sub_cnt = dm->batch - s * per < per ? dm->batch - s * per : per;
    if (w.sub_cnt < 0) w.sub_cnt = 0;
    return w;
}

static int window_count(const LtplLattice* lat, const LtplDims* dm) {
    int n = lat->n_sub;
    while (n > 1 && (dm->batch + n - 1) / n < lat->sub_min) --n;
    if (n > dm->batch) n = dm->batch;
    return n < 1 ? 1 : n;
}

extern "C++" {
template <class Body>
static int for_windows(const LtplLattice* lat, const LtplDims* dm, cudaStream_t st, Body body) {
    const int n = window_count(lat, dm);
    if (n == 1) {
        const LtplDims w = window_dims(dm, 0, 1);
        return body(&w, st);
    }
    if (cudaEventRecord(lat->ev_fork, st) != cudaSuccess) return fail("event record (fork) failed");
    int rc = 0;
    {
        const LtplDims w = window_dims(dm, 0, n);
        rc = body(&w, st);
    }
    int forked = 0;
    for (int s = 1; s < n && rc == 0; ++s, ++forked) {
        cudaStream_t a = lat->aux[s - 1];
        if (cudaStreamWaitEvent(a, lat->ev_fork, 0) != cudaSuccess) {
            rc = fail("stream wait (fork) failed");
            break;
        }
        const LtplDims w = window_dims(dm, s, n);
        const int r = (w.sub_cnt > 0) ? body(&w, a) : 0;
        if (cudaEventRecord(lat->ev_join[s - 1], a) != cudaSuccess && r == 0) rc = fail("event record (join) failed");
        if (r) rc = r;
    }
    for (int s = 1; s <= forked; ++s)   // join whatever was forked, also after an error
        if (cudaStreamWaitEvent(st, lat->ev_join[s - 1], 0) != cudaSuccess && rc == 0) rc = fail("stream wait (join) failed");
    return rc;
}
}  // extern "C++"

// every condition a call of the tick protocol checks; `stateful`: a tick with the iterative memory (ltpl_next_*)
static int validate(const LtplLattice* lat, const LtplParams* prm, const LtplDims* dm, const LtplBuffers* bf,
                    bool stateful) {
    if (!lat || !prm || !dm || !bf) return fail("null argument");
    if (dm->batch <= 0) return fail("dims.batch must be > 0");
    {   // every buffer in front of the optional block (zones, emergency, predictions) is required
        const void* const* ptr = reinterpret_cast<const void* const*>(bf);
        for (size_t i = 0; i < offsetof(LtplBuffers, zone_bits) / sizeof(void*); ++i)
            if (!ptr[i]) return fail("buffers: a required device pointer is NULL");
    }
    if (dm->h_max < 3 || dm->p0_max < 2 || dm->n_export < 1) return fail("dims: h_max >= 3, p0_max >= 2, n_export >= 1");
    if (dm->k_obj < 1) return fail("dims.k_obj must be >= 1");
    {   // (a lattice window too large for any object slot is refused by the k_plan launch)
        const int kmax = max_objects(&lat->h, dm->h_max);
        if (kmax >= 1 && dm->k_obj > kmax) {
            char msg[160];
            snprintf(msg, sizeof(msg), "dims.k_obj: too many object slots for k_plan's shared memory (%d > %d on this "
                     "lattice at h_max %d)", dm->k_obj, kmax, dm->h_max);
            return fail(msg);
        }
    }
    if (dm->p_max % 4 != 0 || dm->p_max < dm->p0_max) return fail("dims.p_max must be a multiple of 4 and >= p0_max");
    if (prm->n_axm < 1 || prm->n_axm > LTPL_MAX_AXM) return fail("params.n_axm out of range");
    if (dm->k_pred < 0 || (dm->k_pred > 0 && (!bf->obj_pred || !bf->n_pred)))
        return fail("dims.k_pred > 0 needs buffers.obj_pred and buffers.n_pred");
    if (dm->n_zones < 0 || (dm->n_zones > 0 && (!bf->zone_bits || !bf->zone_sel || dm->n_zone_words < 1)))
        return fail("dims.n_zones > 0 needs buffers.zone_bits, buffers.zone_sel and dims.n_zone_words");
    if (prm->axm_v[prm->n_axm - 1] < prm->vel_max)  // tph.calc_vel_profile input check
        return fail("ax_max_machines has to cover the entire velocity range of the car (i.e. >= v_max)!");
    if (prm->filt_window < 0 || (prm->filt_window > 1 && prm->filt_window % 2 == 0))   // tph.conv_filt input check
        return fail("params.filt_window: window width of moving average filter must be odd (0 or 1: no smoothing)");
    if (prm->incl_emerg_traj && !bf->em_info) return fail("params.incl_emerg_traj needs buffers.em_info");
    if (!stateful) return 0;
    if (!bf->prev_path || !bf->prev_path_len || !bf->prev_node_idx || !bf->prev_nodes || !bf->prev_n_nodes ||
        !bf->prev_coeff || !bf->prev_s_vx_ax || !bf->prev_action_id || !bf->prev_traj_len || !bf->prev_trim ||
        !bf->sel_action || !bf->pos_last || !bf->t_const || !bf->st_info || !bf->trim || !bf->vel_plan || !bf->course ||
        !bf->obj_dist)
        return fail("stateful tick: the buffers prev_*, sel_action, pos_last, t_const, st_info, trim, vel_plan, course, "
                    "obj_dist must be set");
    if (dm->n_zones > 0 && !bf->zone_s0) return fail("stateful tick with zones: buffers.zone_s0 must be set");
    if (prm->delaycomp <= 0.0) return fail("params.delaycomp must be > 0");
    return 0;
}

int ltpl_set_startpos_batch(const LtplLattice* lat, const LtplParams* prm, const LtplDims* dm, const LtplBuffers* bf,
                            void* stream) {
    if (int r = validate(lat, prm, dm, bf, false)) return r;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    // a new session on a buffer set with memory: its first tick processes the zones anew (GLNT:43-77)
    if (bf->trim && bf->zone_s0 && cudaMemsetAsync(bf->zone_s0, 0xFF, sizeof(int) * (size_t)dm->batch, st) != cudaSuccess)
        return fail("memset(zone_s0) failed");
    k_startpos<<<ctas(dm->batch), kThreads, 0, st>>>(lat->d, *prm, *dm, *bf, 0);
    return check_launch("k_startpos");
}

// buffers.queue_cnt: the path stage starts every count at 0, the velocity stage the export count [2]
static int reset_counts(const LtplBuffers* bf, bool paths, cudaStream_t st) {
    const size_t n = paths ? 4 + 4 * LTPL_MAX_SUB : 1;
    if (cudaMemsetAsync(paths ? bf->queue_cnt : bf->queue_cnt + 2, 0, n * sizeof(int), st) != cudaSuccess)
        return fail("memset(queue_cnt) failed");
    return 0;
}

static int launch_export(const LtplDims* w, const LtplBuffers* bf, cudaStream_t st) {
    k_export<<<ctas(LTPL_NSLOT * w->sub_cnt, LTPL_WARPS_PER_CTA_EXPORT), LTPL_WARPS_PER_CTA_EXPORT * 32, 0, st>>>(*w, *bf);
    return check_launch("k_export");
}

static int launch_emergency(const LtplParams* prm, const LtplDims* w, const LtplBuffers* bf, cudaStream_t st) {
    const size_t smem = emerg_smem_bytes_per_warp(w->n_export) * LTPL_WARPS_PER_CTA;
    if (smem > 48 * 1024) return fail("n_export too large for k_emergency");
    k_emergency<<<ctas(w->sub_cnt), kThreads, smem, st>>>(*prm, *w, *bf);
    return check_launch("k_emergency");
}

// velocity smoothing of every kept profile (params.filt_window > 1); a first tick also rewrites vx, ax of its export rows
static int launch_smooth(const LtplParams* prm, const LtplDims* w, const LtplBuffers* bf, cudaStream_t st, bool stateful) {
    const size_t smem = smooth_smem_bytes_per_warp(w->p_max) * LTPL_WARPS_PER_CTA;
    if (smem > 48 * 1024) return fail("dims.p_max too large for k_smooth");
    k_smooth<<<ctas(LTPL_NSLOT * w->sub_cnt), kThreads, smem, st>>>(*w, *bf, prm->filt_window, stateful ? 0 : 1);
    return check_launch("k_smooth");
}

// one scenario window of calc_paths: (k_startpos of the restarted scenarios -> k_state ->) k_plan -> k_path
static int paths_window(const LtplLattice* lat, const LtplParams* prm, const LtplDims* w, const LtplBuffers* bf,
                        cudaStream_t st, bool stateful) {
    if (stateful && bf->restart) {
        k_startpos<<<ctas(w->sub_cnt), kThreads, 0, st>>>(lat->d, *prm, *w, *bf, 1);
        if (int r = check_launch("k_startpos")) return r;
    }
    if (stateful) {
        k_state<<<ctas(w->sub_cnt), kThreads, 0, st>>>(lat->d, *prm, *w, *bf);
        if (int r = check_launch("k_state")) return r;
    }
    if (int r = launch_k_plan(lat, prm, w, bf, st, stateful)) return r;
    return launch_k_path(lat, prm, w, bf, st, stateful);
}

// one scenario window of calc_vel_profile.  First tick: k_vel_res (exports its rows itself) (-> k_smooth) (-> k_emergency).
// Stateful tick: k_ref -> k_vel_res -> k_backup -> k_prefix (-> k_smooth) -> k_export (-> k_emergency)
static int vel_window(const LtplLattice* lat, const LtplParams* prm, const LtplDims* w, const LtplBuffers* bf,
                      cudaStream_t st, bool stateful) {
    const bool smooth = prm->filt_window > 1;
    if (stateful) {
        k_ref<<<ctas(w->sub_cnt), kThreads, 0, st>>>(lat->d, *prm, *w, *bf);
        if (int r = check_launch("k_ref")) return r;
    }
    if (int r = launch_k_vel(lat, prm, w, bf, st, stateful)) return r;
    if (stateful) {
        k_backup<<<ctas(w->sub_cnt), kThreads, 0, st>>>(*prm, *w, *bf);
        if (int r = check_launch("k_backup")) return r;
        k_prefix<<<ctas(LTPL_NSLOT * w->sub_cnt), kThreads, 0, st>>>(*w, *bf);
        if (int r = check_launch("k_prefix")) return r;
    }
    if (smooth)
        if (int r = launch_smooth(prm, w, bf, st, stateful)) return r;
    if (stateful)
        if (int r = launch_export(w, bf, st)) return r;
    if (prm->incl_emerg_traj) return launch_emergency(prm, w, bf, st);
    return 0;
}

enum { kPaths = 1, kVel = 2 };

// The tick protocol: the stages `stages` (calc_paths, calc_vel_profile or both) of a first tick or of a stateful tick.
// The resets go first, on the caller's stream; then every scenario window runs its whole chain on its stream, one fork /
// join.  A buffer set with memory (trim != NULL) gets the resets of a session: a first tick exports from point 0 (trim
// = 0), and a tick without an emergency trajectory leaves em_info at -1, so that the next stateful tick cannot take a
// stale one for the executed one (k_state).
static int run_tick(const LtplLattice* lat, const LtplParams* prm, const LtplDims* dm, const LtplBuffers* bf,
                    void* stream, int stages, bool stateful) {
    if (int r = validate(lat, prm, dm, bf, stateful)) return r;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const bool paths = stages & kPaths, vel = stages & kVel, memory = bf->trim != nullptr;
    const size_t B = dm->batch;
    if (int r = reset_counts(bf, paths, st)) return r;
    if (memory && paths && !stateful && cudaMemsetAsync(bf->trim, 0, sizeof(int) * 4 * LTPL_NSLOT * B, st) != cudaSuccess)
        return fail("memset(trim) failed");
    if (memory && vel && !prm->incl_emerg_traj && bf->em_info &&
        cudaMemsetAsync(bf->em_info, 0xFF, sizeof(int) * 3 * B, st) != cudaSuccess)
        return fail("memset(em_info) failed");
    // `vel` is the start velocity of set_startpos (k_state reads it); the velocity stages of a stateful tick start at the
    // planned velocity at the cut instead
    LtplBuffers vbf = *bf;
    if (stateful) vbf.vel = bf->vel_plan;
    return for_windows(lat, dm, st, [&](const LtplDims* w, cudaStream_t s) {
        if (paths)
            if (int r = paths_window(lat, prm, w, bf, s, stateful)) return r;
        return vel ? vel_window(lat, prm, w, &vbf, s, stateful) : 0;
    });
}

int ltpl_calc_paths_batch(const LtplLattice* lat, const LtplParams* prm, const LtplDims* dm, const LtplBuffers* bf,
                          void* stream) {
    return run_tick(lat, prm, dm, bf, stream, kPaths, false);
}

int ltpl_calc_vel_profile_batch(const LtplLattice* lat, const LtplParams* prm, const LtplDims* dm,
                                const LtplBuffers* bf, void* stream) {
    return run_tick(lat, prm, dm, bf, stream, kVel, false);
}

int ltpl_tick_batch(const LtplLattice* lat, const LtplParams* prm, const LtplDims* dm, const LtplBuffers* bf,
                    void* stream) {
    return run_tick(lat, prm, dm, bf, stream, kPaths | kVel, false);
}

// stateful tick (ltpl_state.cuh):
//   ltpl_next_calc_paths_batch        (k_startpos masked by buffers.restart ->) k_state -> k_plan<.., true> -> k_path<true>
//   ltpl_next_calc_vel_profile_batch  k_ref -> k_vel_res<true> -> k_backup -> k_prefix -> k_export
int ltpl_next_calc_paths_batch(const LtplLattice* lat, const LtplParams* prm, const LtplDims* dm, const LtplBuffers* bf,
                               void* stream) {
    return run_tick(lat, prm, dm, bf, stream, kPaths, true);
}

int ltpl_next_calc_vel_profile_batch(const LtplLattice* lat, const LtplParams* prm, const LtplDims* dm,
                                     const LtplBuffers* bf, void* stream) {
    return run_tick(lat, prm, dm, bf, stream, kVel, true);
}

int ltpl_next_tick_batch(const LtplLattice* lat, const LtplParams* prm, const LtplDims* dm, const LtplBuffers* bf,
                         void* stream) {
    return run_tick(lat, prm, dm, bf, stream, kPaths | kVel, true);
}

int ltpl_launch_stage(int stage, const LtplLattice* lat, const LtplParams* prm, const LtplDims* dm,
                      const LtplBuffers* bf, void* stream) {
    if (int r = validate(lat, prm, dm, bf, false)) return r;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const LtplDims w = window_dims(dm, 0, 1);   // the whole batch as ONE window: this call times a kernel alone
    switch (stage) {
        case 0: return ltpl_set_startpos_batch(lat, prm, dm, bf, stream);
        case 1: return launch_k_plan(lat, prm, &w, bf, st, false);
        case 2:
            if (int r = reset_counts(bf, true, st)) return r;
            return launch_k_path(lat, prm, &w, bf, st, false);
        case 3:
            if (int r = reset_counts(bf, false, st)) return r;
            return launch_k_vel(lat, prm, &w, bf, st, false);
        case 4: return launch_export(&w, bf, st);
        default: return fail("ltpl_launch_stage: unknown stage");
    }
}

int ltpl_velprofile_batch(const LtplParams* prm, const LtplVelBatch* vb, void* stream) {
    if (!prm || !vb) return fail("null argument");
    if (vb->n_paths <= 0 || vb->n_points < 2) return fail("velprofile: need n_paths > 0 and n_points >= 2");
    if (prm->n_axm < 1 || prm->n_axm > LTPL_MAX_AXM) return fail("params.n_axm out of range");
    if (prm->axm_v[prm->n_axm - 1] < prm->vel_max)
        return fail("ax_max_machines has to cover the entire velocity range of the car (i.e. >= v_max)!");
    if (prm->dyn_model_exp == 1.0)
        k_velprofile<true><<<(vb->n_paths + 31) / 32, 32, VD_SMEM_BYTES, static_cast<cudaStream_t>(stream)>>>(*prm, *vb);
    else
        k_velprofile<false><<<(vb->n_paths + 31) / 32, 32, VD_SMEM_BYTES, static_cast<cudaStream_t>(stream)>>>(*prm, *vb);
    return check_launch("k_velprofile");
}

#ifdef LTPL_PROFILE_PHASES
int ltpl_debug_phases(unsigned long long* out32, int reset) {
    if (out32) cudaMemcpyFromSymbol(out32, g_phase, sizeof(unsigned long long) * 32);
    if (reset) {
        unsigned long long z[32] = {0};
        cudaMemcpyToSymbol(g_phase, z, sizeof(z));
    }
    return 0;
}
#endif

}  // extern "C"
