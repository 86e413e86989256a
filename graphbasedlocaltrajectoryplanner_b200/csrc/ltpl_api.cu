// ltpl_api.cu -- C-ABI of libltpl_b200.so (include/ltpl_b200.h).  Host side only resolves pointers and launches
// kernels on the caller's stream; no allocation, no synchronisation on the hot path.
//
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -fmad=false -shared -Xcompiler -fPIC
#include <atomic>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>

#define LTPL_WARPS_PER_CTA_EXPORT 8
#include "ltpl_path.cuh"
#include "ltpl_plan.cuh"
#include "ltpl_vel.cuh"
#include "ltpl_vel_res.cuh"
#include "ltpl_velprofile.cuh"
#include "ltpl_emerg.cuh"
#include "ltpl_state.cuh"
#include "ltpl_smooth.cuh"

static std::atomic<unsigned long long> g_launches{0};

// velocity kernel: one CTA per VR_P queued paths of one class, the paths resident in shared memory (ltpl_vel_res.cuh)
static cudaError_t launch_k_vel(const LtplLattice* lat, const LtplParams* prm, const LtplDims* dm, const LtplBuffers* bf,
                                cudaStream_t st, bool stateful = false) {
    const int nq = LTPL_NSLOT * dm->sub_cnt;   // paths of this launch's scenario window
    const int nmax = dm->p_max;
    if (nmax > 32 * VR_MAXM || nmax % 4 != 0) return cudaErrorInvalidValue;
    const bool gg = bf->gg != nullptr;   // location dependent local_gg: the general-exponent variant carries it
    const size_t smem = vr_smem_bytes(nmax, gg);
    if (smem > 200 * 1024) return cudaErrorInvalidValue;
    static thread_local size_t attr_set = 0;
    if (smem > attr_set) {
        const void* fns[6] = {(const void*)k_vel_res<false, true, false>, (const void*)k_vel_res<true, true, false>,
                              (const void*)k_vel_res<false, false, false>, (const void*)k_vel_res<true, false, false>,
                              (const void*)k_vel_res<false, false, true>, (const void*)k_vel_res<true, false, true>};
        for (const void* f : fns)
            if (cudaError_t e = cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) return e;
        attr_set = smem;
    }
    const int grid = nq / VR_P + 2;   // >= groups of the follow queue + groups of the other queue
    const bool exp1 = prm->dyn_model_exp == 1.0 && !gg;
    if (gg && stateful)
        k_vel_res<true, false, true><<<grid, VR_THREADS, smem, st>>>(lat->d, *prm, *dm, *bf, nmax);
    else if (gg)
        k_vel_res<false, false, true><<<grid, VR_THREADS, smem, st>>>(lat->d, *prm, *dm, *bf, nmax);
    else if (stateful && exp1)
        k_vel_res<true, true, false><<<grid, VR_THREADS, smem, st>>>(lat->d, *prm, *dm, *bf, nmax);
    else if (stateful)
        k_vel_res<true, false, false><<<grid, VR_THREADS, smem, st>>>(lat->d, *prm, *dm, *bf, nmax);
    else if (exp1)
        k_vel_res<false, true, false><<<grid, VR_THREADS, smem, st>>>(lat->d, *prm, *dm, *bf, nmax);
    else
        k_vel_res<false, false, false><<<grid, VR_THREADS, smem, st>>>(lat->d, *prm, *dm, *bf, nmax);
    return cudaSuccess;
}

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


// k_plan<ZONE, STATE>: one warp per scenario (ltpl_plan.cuh)
static const char* launch_k_plan(const LtplLattice* lat, const LtplParams* prm, const LtplDims* dm, const LtplBuffers* bf,
                                 cudaStream_t st, bool stateful) {
    const int maxn = ((lat->h.max_nodes_per_layer + 31) / 32) * 32;
    const int hl = dm->h_max;
    const int mask_words = (lat->h.max_window_edges + 31) / 32 + 1;
    const size_t smem = plan_smem_bytes_per_warp(maxn, hl, mask_words) * LTPL_WARPS_PER_CTA;
    if (smem > 200 * 1024) return "lattice window too large for shared memory";
    const bool zone = dm->n_zones > 0;
    const bool dense = lat->h.num_edges >= 2 * lat->h.num_nodes;   // in-edges per node (dp_run<.., DENSE>)
    typedef void (*PlanFn)(const __grid_constant__ LatDev, const __grid_constant__ LtplParams, const __grid_constant__ LtplDims,
                           const __grid_constant__ LtplBuffers, const int, const int, const int);
    static const PlanFn fns[8] = {k_plan<false, false, false>, k_plan<true, false, false>, k_plan<false, true, false>,
                                  k_plan<true, true, false>,   k_plan<false, false, true>, k_plan<true, false, true>,
                                  k_plan<false, true, true>,   k_plan<true, true, true>};
    static thread_local size_t attr = 0;
    if (smem > 48 * 1024 && smem > attr) {
        for (PlanFn f : fns)
            if (cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
                return "cudaFuncSetAttribute(k_plan) failed";
        attr = smem;
    }
    const int grid = (dm->sub_cnt + LTPL_WARPS_PER_CTA - 1) / LTPL_WARPS_PER_CTA, thr = LTPL_WARPS_PER_CTA * 32;
    fns[(zone ? 1 : 0) + (stateful ? 2 : 0) + (dense ? 4 : 0)]<<<grid, thr, smem, st>>>(lat->d, *prm, *dm, *bf, maxn, hl,
                                                                                        mask_words);
    return nullptr;
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
        cudaError_t e = cudaSuccess;
        if (smem > 200 * 1024) {
            delete lat;
            return fail("ltpl_lattice_create: planning range too large for shared memory");
        }
        if (smem > 48 * 1024)
            e = cudaFuncSetAttribute(k_follow_table, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e == cudaSuccess) {
            k_follow_table<<<(h->num_nodes + LTPL_WARPS_PER_CTA - 1) / LTPL_WARPS_PER_CTA, LTPL_WARPS_PER_CTA * 32, smem>>>(
                d, maxn, reinterpret_cast<int*>(p + h->off_tab_reach), p + h->off_tab_node,
                reinterpret_cast<int*>(p + h->off_tab_edge));
            e = cudaGetLastError();
        }
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

static int check_common(const LtplLattice* lat, const LtplParams* prm, const LtplDims* dm, const LtplBuffers* bf) {
    if (!lat || !prm || !dm || !bf) return fail("null argument");
    if (dm->batch <= 0) return fail("dims.batch must be > 0");
    {   // every buffer in front of the optional block (zones, emergency, predictions) is required
        const void* const* ptr = reinterpret_cast<const void* const*>(bf);
        for (size_t i = 0; i < offsetof(LtplBuffers, zone_bits) / sizeof(void*); ++i)
            if (!ptr[i]) return fail("buffers: a required device pointer is NULL");
    }
    if (dm->h_max < 3 || dm->p0_max < 2 || dm->n_export < 1) return fail("dims: h_max >= 3, p0_max >= 2, n_export >= 1");
    if (dm->k_obj < 1 || dm->k_obj > LTPL_KMAX) return fail("dims.k_obj must be in [1, 16]");
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
    return 0;
}

int ltpl_set_startpos_batch(const LtplLattice* lat, const LtplParams* prm, const LtplDims* dm, const LtplBuffers* bf,
                            void* stream) {
    if (int r = check_common(lat, prm, dm, bf)) return r;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int grid = (dm->batch + LTPL_WARPS_PER_CTA - 1) / LTPL_WARPS_PER_CTA;
    k_startpos<<<grid, LTPL_WARPS_PER_CTA * 32, 0, st>>>(lat->d, *prm, *dm, *bf);
    return check_launch("k_startpos");
}

static const int kCntInts = 4 + 4 * LTPL_MAX_SUB;   // buffers.queue_cnt

static int prepare_path_attr(const LtplDims* dm, bool stateful, size_t* smem_out) {
    const size_t smem_path = path_smem_bytes_per_warp(dm->h_max) * LTPL_WARPS_PER_CTA;
    if (smem_path > 200 * 1024) return fail("lattice window too large for shared memory");
    static thread_local size_t attr_path[2] = {0, 0};
    if (smem_path > 48 * 1024 && smem_path > attr_path[stateful]) {
        const cudaError_t e = stateful ? cudaFuncSetAttribute(k_path<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_path)
                                       : cudaFuncSetAttribute(k_path<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_path);
        if (e != cudaSuccess) return fail("cudaFuncSetAttribute(k_path) failed");
        attr_path[stateful] = smem_path;
    }
    *smem_out = smem_path;
    return 0;
}

// one scenario window of calc_paths: (k_state ->) k_plan -> k_path
static int paths_window(const LtplLattice* lat, const LtplParams* prm, const LtplDims* w, const LtplBuffers* bf,
                        cudaStream_t st, bool stateful, size_t smem_path) {
    const int grid_b = (w->sub_cnt + LTPL_WARPS_PER_CTA - 1) / LTPL_WARPS_PER_CTA;
    const int grid_q = (LTPL_NSLOT * w->sub_cnt + LTPL_WARPS_PER_CTA - 1) / LTPL_WARPS_PER_CTA;
    if (stateful) {
        k_state<<<grid_b, LTPL_WARPS_PER_CTA * 32, 0, st>>>(lat->d, *prm, *w, *bf);
        if (int r = check_launch("k_state")) return r;
    }
    if (const char* e = launch_k_plan(lat, prm, w, bf, st, stateful)) return fail(e);
    if (int r = check_launch("k_plan")) return r;
    if (stateful)
        k_path<true><<<grid_q, LTPL_WARPS_PER_CTA * 32, smem_path, st>>>(lat->d, *prm, *w, *bf);
    else
        k_path<false><<<grid_q, LTPL_WARPS_PER_CTA * 32, smem_path, st>>>(lat->d, *prm, *w, *bf);
    return check_launch("k_path");
}

static int launch_emergency(const LtplParams* prm, const LtplDims* w, const LtplBuffers* bf, cudaStream_t st) {
    const size_t smem = emerg_smem_bytes_per_warp(w->n_export) * LTPL_WARPS_PER_CTA;
    if (smem > 48 * 1024) return fail("n_export too large for k_emergency");
    k_emergency<<<(w->sub_cnt + LTPL_WARPS_PER_CTA - 1) / LTPL_WARPS_PER_CTA, LTPL_WARPS_PER_CTA * 32, smem, st>>>(
        *prm, *w, *bf);
    return check_launch("k_emergency");
}

static const char* kVelCapacity =
    "k_vel: dims.p_max exceeds the shared-memory capacity of the velocity kernel (<= 512, % 4 == 0)";

// velocity smoothing of every kept profile (params.filt_window > 1); a first tick also rewrites vx, ax of its export rows
static int launch_smooth(const LtplParams* prm, const LtplDims* w, const LtplBuffers* bf, cudaStream_t st, bool stateful) {
    const size_t smem = smooth_smem_bytes_per_warp(w->p_max) * LTPL_WARPS_PER_CTA;
    if (smem > 48 * 1024) return fail("dims.p_max too large for k_smooth");
    const int nq = LTPL_NSLOT * w->sub_cnt;
    k_smooth<<<(nq + LTPL_WARPS_PER_CTA - 1) / LTPL_WARPS_PER_CTA, LTPL_WARPS_PER_CTA * 32, smem, st>>>(
        *w, *bf, prm->filt_window, stateful ? 0 : 1);
    return check_launch("k_smooth");
}

// one scenario window of calc_vel_profile.  First tick: k_vel_res (exports its rows itself) (-> k_smooth) (-> k_emergency).
// Stateful tick: k_ref -> k_vel_res -> k_backup -> k_prefix (-> k_smooth) -> k_export (-> k_emergency)
static int vel_window(const LtplLattice* lat, const LtplParams* prm, const LtplDims* w, const LtplBuffers* bf,
                      cudaStream_t st, bool stateful) {
    const bool smooth = prm->filt_window > 1;
    const int grid_b = (w->sub_cnt + LTPL_WARPS_PER_CTA - 1) / LTPL_WARPS_PER_CTA;
    const int nq = LTPL_NSLOT * w->sub_cnt;
    const int grid_q = (nq + LTPL_WARPS_PER_CTA - 1) / LTPL_WARPS_PER_CTA;
    if (stateful) {
        k_ref<<<grid_b, LTPL_WARPS_PER_CTA * 32, 0, st>>>(lat->d, *prm, *w, *bf);
        if (int r = check_launch("k_ref")) return r;
    }
    if (launch_k_vel(lat, prm, w, bf, st, stateful) != cudaSuccess) return fail(kVelCapacity);
    if (int r = check_launch("k_vel")) return r;
    if (stateful) {
        k_backup<<<grid_b, LTPL_WARPS_PER_CTA * 32, 0, st>>>(*prm, *w, *bf);
        if (int r = check_launch("k_backup")) return r;
        k_prefix<<<grid_q, LTPL_WARPS_PER_CTA * 32, 0, st>>>(*w, *bf);
        if (int r = check_launch("k_prefix")) return r;
        if (smooth)
            if (int r = launch_smooth(prm, w, bf, st, true)) return r;
        k_export<<<(nq + LTPL_WARPS_PER_CTA_EXPORT - 1) / LTPL_WARPS_PER_CTA_EXPORT, LTPL_WARPS_PER_CTA_EXPORT * 32, 0,
                   st>>>(*w, *bf);
        if (int r = check_launch("k_export")) return r;
    } else if (smooth) {
        if (int r = launch_smooth(prm, w, bf, st, false)) return r;
    }
    if (prm->incl_emerg_traj) return launch_emergency(prm, w, bf, st);
    return 0;
}

static int launch_paths(const LtplLattice* lat, const LtplParams* prm, const LtplDims* dm, const LtplBuffers* bf,
                        cudaStream_t st, bool stateful) {
    size_t smem_path = 0;
    if (int r = prepare_path_attr(dm, stateful, &smem_path)) return r;
    if (cudaMemsetAsync(bf->queue_cnt, 0, kCntInts * sizeof(int), st) != cudaSuccess) return fail("memset(queue_cnt) failed");
    return for_windows(lat, dm, st, [&](const LtplDims* w, cudaStream_t s) {
        return paths_window(lat, prm, w, bf, s, stateful, smem_path);
    });
}

static int launch_vel(const LtplLattice* lat, const LtplParams* prm, const LtplDims* dm, const LtplBuffers* bf,
                      cudaStream_t st, bool stateful) {
    if (prm->incl_emerg_traj && !bf->em_info) return fail("params.incl_emerg_traj needs buffers.em_info");
    if (cudaMemsetAsync(bf->queue_cnt + 2, 0, sizeof(int), st) != cudaSuccess) return fail("memset(export count) failed");
    if (int r = for_windows(lat, dm, st, [&](const LtplDims* w, cudaStream_t s) {
            return vel_window(lat, prm, w, bf, s, stateful);
        }))
        return r;
    // stateful tick without an emergency trajectory: the next one must not take a stale one for executed (k_state)
    if (stateful && !prm->incl_emerg_traj && bf->em_info &&
        cudaMemsetAsync(bf->em_info, 0xFF, sizeof(int) * 3 * (size_t)dm->batch, st) != cudaSuccess)
        return fail("memset(em_info) failed");
    return 0;
}

// calc_paths + calc_vel_profile of one tick: every window runs its whole chain on its stream, one fork / join
static int launch_tick(const LtplLattice* lat, const LtplParams* prm, const LtplDims* dm, const LtplBuffers* bf,
                       cudaStream_t st, bool stateful) {
    size_t smem_path = 0;
    if (int r = prepare_path_attr(dm, stateful, &smem_path)) return r;
    if (prm->incl_emerg_traj && !bf->em_info) return fail("params.incl_emerg_traj needs buffers.em_info");
    if (cudaMemsetAsync(bf->queue_cnt, 0, kCntInts * sizeof(int), st) != cudaSuccess) return fail("memset(queue_cnt) failed");
    if (int r = for_windows(lat, dm, st, [&](const LtplDims* w, cudaStream_t s) {
            if (int r2 = paths_window(lat, prm, w, bf, s, stateful, smem_path)) return r2;
            return vel_window(lat, prm, w, bf, s, stateful);
        }))
        return r;
    if (stateful && !prm->incl_emerg_traj && bf->em_info &&
        cudaMemsetAsync(bf->em_info, 0xFF, sizeof(int) * 3 * (size_t)dm->batch, st) != cudaSuccess)
        return fail("memset(em_info) failed");
    return 0;
}

int ltpl_calc_paths_batch(const LtplLattice* lat, const LtplParams* prm, const LtplDims* dm, const LtplBuffers* bf,
                          void* stream) {
    if (int r = check_common(lat, prm, dm, bf)) return r;
    return launch_paths(lat, prm, dm, bf, static_cast<cudaStream_t>(stream), false);
}

int ltpl_calc_vel_profile_batch(const LtplLattice* lat, const LtplParams* prm, const LtplDims* dm,
                                const LtplBuffers* bf, void* stream) {
    if (int r = check_common(lat, prm, dm, bf)) return r;
    return launch_vel(lat, prm, dm, bf, static_cast<cudaStream_t>(stream), false);
}

int ltpl_tick_batch(const LtplLattice* lat, const LtplParams* prm, const LtplDims* dm, const LtplBuffers* bf,
                    void* stream) {
    if (int r = check_common(lat, prm, dm, bf)) return r;
    return launch_tick(lat, prm, dm, bf, static_cast<cudaStream_t>(stream), false);
}

// stateful tick (ltpl_state.cuh):
//   ltpl_next_calc_paths_batch        k_state -> k_plan<.., true> -> k_path<true>
//   ltpl_next_calc_vel_profile_batch  k_ref -> k_vel_res<true> -> k_backup -> k_prefix -> k_export
static int check_stateful(const LtplLattice* lat, const LtplParams* prm, const LtplDims* dm, const LtplBuffers* bf) {
    if (int r = check_common(lat, prm, dm, bf)) return r;
    if (!bf->prev_path || !bf->prev_path_len || !bf->prev_node_idx || !bf->prev_nodes || !bf->prev_n_nodes ||
        !bf->prev_coeff || !bf->prev_s_vx_ax || !bf->prev_action_id || !bf->prev_traj_len || !bf->prev_trim ||
        !bf->sel_action || !bf->pos_last || !bf->t_const || !bf->st_info || !bf->trim || !bf->vel_plan || !bf->course ||
        !bf->obj_dist)
        return fail("stateful tick: the buffers prev_*, sel_action, pos_last, t_const, st_info, trim, vel_plan, course, "
                    "obj_dist must be set");
    if (dm->n_zones > 0 && !bf->zone_s0) return fail("stateful tick with zones: buffers.zone_s0 must be set");
    if (prm->incl_emerg_traj && !bf->em_info) return fail("params.incl_emerg_traj needs buffers.em_info");
    if (prm->delaycomp <= 0.0) return fail("params.delaycomp must be > 0");
    return 0;
}

int ltpl_next_calc_paths_batch(const LtplLattice* lat, const LtplParams* prm, const LtplDims* dm, const LtplBuffers* bf,
                               void* stream) {
    if (int r = check_stateful(lat, prm, dm, bf)) return r;
    return launch_paths(lat, prm, dm, bf, static_cast<cudaStream_t>(stream), true);
}

int ltpl_next_calc_vel_profile_batch(const LtplLattice* lat, const LtplParams* prm, const LtplDims* dm,
                                     const LtplBuffers* bf, void* stream) {
    if (int r = check_stateful(lat, prm, dm, bf)) return r;
    if (bf->vel != bf->vel_plan) return fail("stateful tick: buffers.vel must point at buffers.vel_plan");
    return launch_vel(lat, prm, dm, bf, static_cast<cudaStream_t>(stream), true);
}

int ltpl_next_tick_batch(const LtplLattice* lat, const LtplParams* prm, const LtplDims* dm, const LtplBuffers* bf,
                         void* stream) {
    if (int r = check_stateful(lat, prm, dm, bf)) return r;
    if (bf->vel != bf->vel_plan) return fail("stateful tick: buffers.vel must point at buffers.vel_plan");
    return launch_tick(lat, prm, dm, bf, static_cast<cudaStream_t>(stream), true);
}

int ltpl_launch_stage(int stage, const LtplLattice* lat, const LtplParams* prm, const LtplDims* dm,
                      const LtplBuffers* bf, void* stream) {
    if (int r = check_common(lat, prm, dm, bf)) return r;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const LtplDims w = window_dims(dm, 0, 1);   // the whole batch as ONE window: this call times a kernel alone
    const int nq = LTPL_NSLOT * dm->batch;
    switch (stage) {
        case 0: return ltpl_set_startpos_batch(lat, prm, dm, bf, stream);
        case 1:
            if (const char* e = launch_k_plan(lat, prm, &w, bf, st, false)) return fail(e);
            return check_launch("k_plan");
        case 2: {
            size_t smem_path = 0;
            if (int r = prepare_path_attr(dm, false, &smem_path)) return r;
            if (cudaMemsetAsync(bf->queue_cnt, 0, kCntInts * sizeof(int), st) != cudaSuccess)
                return fail("memset(queue_cnt) failed");
            k_path<false><<<(nq + LTPL_WARPS_PER_CTA - 1) / LTPL_WARPS_PER_CTA, LTPL_WARPS_PER_CTA * 32, smem_path, st>>>(
                lat->d, *prm, w, *bf);
            return check_launch("k_path");
        }
        case 3:
            if (cudaMemsetAsync(bf->queue_cnt + 2, 0, sizeof(int), st) != cudaSuccess)
                return fail("memset(export count) failed");
            if (launch_k_vel(lat, prm, &w, bf, st) != cudaSuccess) return fail(kVelCapacity);
            return check_launch("k_vel");
        case 4:
            k_export<<<(nq + LTPL_WARPS_PER_CTA_EXPORT - 1) / LTPL_WARPS_PER_CTA_EXPORT,
                       LTPL_WARPS_PER_CTA_EXPORT * 32, 0, st>>>(w, *bf);
            return check_launch("k_export");
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
