// ltpl_api.cu -- C-ABI of libltpl_b200.so (include/ltpl_b200.h).  Host side only resolves pointers and launches
// kernels on the caller's stream; no allocation, no synchronisation on the hot path.
//
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -fmad=false -shared -Xcompiler -fPIC
#include <atomic>
#include <cmath>
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
#include "ltpl_velfollow.cuh"
#include "ltpl_emerg.cuh"
#include "ltpl_state.cuh"
#include "ltpl_smooth.cuh"
#include "ltpl_gg_map.cuh"
#include "ltpl_stage.cuh"
#include "ltpl_traj_base.cuh"
#include "ltpl_select.cuh"
#include "ltpl_pathcoord.cuh"

// the memory records are the int32 arrays BatchPlanner allocates: st_info [B][8], trim [NSLOT*B][4]
static_assert(sizeof(LtplStateInfo) == 8 * sizeof(int32_t) && alignof(LtplStateInfo) == alignof(int32_t), "st_info row");
static_assert(offsetof(LtplStateInfo, prev_q) == 0 && offsetof(LtplStateInfo, prev_m) == 4 &&
              offsetof(LtplStateInfo, prev_L) == 8 && offsetof(LtplStateInfo, const_nodes) == 12 &&
              offsetof(LtplStateInfo, n_factored) == 16 && offsetof(LtplStateInfo, factored_edge) == 20, "st_info row");
static_assert(sizeof(LtplTrim) == 4 * sizeof(int32_t) && alignof(LtplTrim) == alignof(int32_t), "trim row");
static_assert(offsetof(LtplTrim, m) == 0 && offsetof(LtplTrim, L) == 4 && offsetof(LtplTrim, cut) == 8 &&
              offsetof(LtplTrim, pref) == 12, "trim row");

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

static size_t plan_smem(const LtplLattice* lat, const LtplDims* dm) {
    return plan_smem_bytes_per_warp(plan_maxn(&lat->h), dm->h_max, plan_mask_words(&lat->h), dm->k_obj) *
           LTPL_WARPS_PER_CTA;
}

// k_plan's attributes for these dims: the dynamic shared-memory limit and the carveout (set when they change)
static int plan_attributes(const LtplLattice* lat, const LtplDims* dm) {
    const int maxn = plan_maxn(&lat->h);
    const int hl = dm->h_max;
    const int mask_words = plan_mask_words(&lat->h);
    if (int r = allow_smem(lat, kSmemPlan, plan_smem(lat, dm), kPlanFns, "k_plan",
                           "lattice window too large for shared memory"))
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
    return 0;
}

static int launch_k_plan(const LtplLattice* lat, const LtplParams* prm, const LtplDims* dm, const LtplBuffers* bf,
                         cudaStream_t st, bool stateful) {
    if (int r = plan_attributes(lat, dm)) return r;
    const int maxn = plan_maxn(&lat->h);
    const int hl = dm->h_max;
    const int mask_words = plan_mask_words(&lat->h);
    const size_t smem = plan_smem(lat, dm);
    const bool zone = dm->n_zones > 0;
    const bool dense = lat->h.num_edges >= 2 * lat->h.num_nodes;   // in-edges per node (dp_run<.., DENSE>)
    kPlanFns[(zone ? 1 : 0) + (stateful ? 2 : 0) + (dense ? 4 : 0)]<<<ctas(dm->sub_cnt), kThreads, smem, st>>>(
        lat->d, *prm, *dm, *bf, maxn, hl, mask_words);
    return check_launch("k_plan");
}

// k_path<STATE>: one warp per path (ltpl_path.cuh)
typedef void (*PathFn)(const __grid_constant__ LatDev, const __grid_constant__ LtplParams, const __grid_constant__ LtplDims,
                       const __grid_constant__ LtplBuffers);
static const PathFn kPathFns[2] = {k_path<false>, k_path<true>};

static size_t path_smem(const LtplDims* dm) { return path_smem_bytes_per_warp(dm->h_max) * LTPL_WARPS_PER_CTA; }

static int path_attributes(const LtplLattice* lat, const LtplDims* dm) {
    return allow_smem(lat, kSmemPath, path_smem(dm), kPathFns, "k_path", "lattice window too large for shared memory");
}

static int launch_k_path(const LtplLattice* lat, const LtplParams* prm, const LtplDims* dm, const LtplBuffers* bf,
                         cudaStream_t st, bool stateful) {
    const size_t smem = path_smem(dm);
    if (int r = path_attributes(lat, dm)) return r;
    kPathFns[stateful]<<<ctas(LTPL_NSLOT * dm->sub_cnt), kThreads, smem, st>>>(lat->d, *prm, *dm, *bf);
    return check_launch("k_path");
}

// velocity kernel: one CTA per VR_P queued paths of one class, the paths resident in shared memory (ltpl_vel_res.cuh)
typedef void (*VelFn)(const LatDev, const LtplParams, const LtplDims, const LtplBuffers, const int);
// <STATE, EXP1, GG>: [stateful + 2 * (0 exponent 1, 1 general exponent, 2 local_gg planes)]
static const VelFn kVelFns[6] = {k_vel_res<false, true, false>, k_vel_res<true, true, false>,
                                 k_vel_res<false, false, false>, k_vel_res<true, false, false>,
                                 k_vel_res<false, false, true>, k_vel_res<true, false, true>};

static int vel_attributes(const LtplLattice* lat, const LtplDims* dm, const LtplBuffers* bf) {
    const int nmax = dm->p_max;
    if (nmax > 32 * VR_MAXM)
        return fail("k_vel: dims.p_max exceeds the shared-memory capacity of the velocity kernel (<= 512)");
    // location dependent local_gg: the general-exponent variant carries it
    return allow_smem(lat, kSmemVel, vr_smem_bytes(nmax, bf->gg != nullptr), kVelFns, "k_vel",
                      "dims.p_max too large for the velocity kernel's shared memory");
}

static int launch_k_vel(const LtplLattice* lat, const LtplParams* prm, const LtplDims* dm, const LtplBuffers* bf,
                        cudaStream_t st, bool stateful) {
    if (int r = vel_attributes(lat, dm, bf)) return r;
    const int nmax = dm->p_max;
    const bool gg = bf->gg != nullptr;
    const size_t smem = vr_smem_bytes(nmax, gg);
    const int kind = gg ? 2 : (prm->dyn_model_exp == 1.0 ? 0 : 1);
    const int nq = LTPL_NSLOT * dm->sub_cnt;   // paths of this launch's scenario window
    const int grid = nq / VR_P + 2;            // >= groups of the follow queue + groups of the other queue
    kVelFns[(stateful ? 1 : 0) + 2 * kind]<<<grid, VR_THREADS, smem, st>>>(lat->d, *prm, *dm, *bf, nmax);
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
        case 5: return (int)sizeof(LtplStageSrc);
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
    if (bf->gg_map) {   // the friction map fills the caller's gg planes (k_gg_map)
        if (!bf->gg) return fail("buffers.gg_map needs buffers.gg: the planes the map is evaluated into");
        if (reinterpret_cast<uintptr_t>(bf->gg_map) % 16 != 0)
            return fail("buffers.gg_map must be 16-byte aligned (k_gg_map reads one ax, ay pair per 16-byte load)");
        if (prm->gg_map_nx < 2 || prm->gg_map_ny < 2) return fail("params.gg_map_nx and params.gg_map_ny must be >= 2");
        if ((int64_t)prm->gg_map_nx * prm->gg_map_ny > INT32_MAX)
            return fail("params.gg_map_nx * params.gg_map_ny exceeds 32-bit indexing");
        if (!std::isfinite(prm->gg_map_inv_cell) || !(prm->gg_map_inv_cell > 0.0))
            return fail("params.gg_map_inv_cell must be finite and > 0");
        if (!std::isfinite(prm->gg_map_x0) || !std::isfinite(prm->gg_map_y0))
            return fail("params.gg_map_x0 and params.gg_map_y0 must be finite");
    }
    if (bf->traj_base) {   // ids from the device counter (k_traj_base)
        if (prm->traj_base_id != 0)
            return fail("buffers.traj_base needs params.traj_base_id = 0: k_traj_base adds the base from the counter");
        if (reinterpret_cast<uintptr_t>(bf->traj_base) % 4 != 0) return fail("buffers.traj_base must be 4-byte aligned");
    }
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

// one scenario window of calc_vel_profile, behind k_gg_map when a friction map is set.  First tick: k_vel_res (exports its
// rows itself) (-> k_smooth) (-> k_emergency).  Stateful tick: k_ref -> k_vel_res -> k_backup -> k_prefix (-> k_smooth) ->
// k_export (-> k_emergency)
static int vel_window(const LtplLattice* lat, const LtplParams* prm, const LtplDims* w, const LtplBuffers* bf,
                      cudaStream_t st, bool stateful) {
    const bool smooth = prm->filt_window > 1;
    if (bf->gg_map) {
        k_gg_map<<<ctas(LTPL_NSLOT * w->sub_cnt), kThreads, 0, st>>>(*prm, *w, *bf);
        if (int r = check_launch("k_gg_map")) return r;
    }
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
    if (memory && paths && !stateful && cudaMemsetAsync(bf->trim, 0, sizeof(LtplTrim) * LTPL_NSLOT * B, st) != cudaSuccess)
        return fail("memset(trim) failed");
    if (memory && vel && !prm->incl_emerg_traj && bf->em_info &&
        cudaMemsetAsync(bf->em_info, 0xFF, sizeof(int) * 3 * B, st) != cudaSuccess)
        return fail("memset(em_info) failed");
    // `vel` is the start velocity of set_startpos (k_state reads it); the velocity stages of a stateful tick start at the
    // planned velocity at the cut instead
    LtplBuffers vbf = *bf;
    if (stateful) vbf.vel = bf->vel_plan;
    if (int r = for_windows(lat, dm, st, [&](const LtplDims* w, cudaStream_t s) {
            if (paths)
                if (int r = paths_window(lat, prm, w, bf, s, stateful)) return r;
            return vel ? vel_window(lat, prm, w, &vbf, s, stateful) : 0;
        }))
        return r;
    if (!vel || !bf->traj_base) return 0;
    // trajectory ids from the device counter, behind the join: every window's ids are written
    k_traj_base<<<1, LTPL_TRAJ_BASE_THREADS, 0, st>>>(bf->traj_base, bf->traj_id, prm->incl_emerg_traj ? bf->em_info : nullptr,
                                                      (int)(LTPL_NSLOT * B), (int)B);
    return check_launch("k_traj_base");
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

int ltpl_prepare_batch(const LtplLattice* lat, const LtplParams* prm, const LtplDims* dm, const LtplBuffers* bf) {
    if (int r = validate(lat, prm, dm, bf, false)) return r;
    if (int r = plan_attributes(lat, dm)) return r;
    if (int r = path_attributes(lat, dm)) return r;
    return vel_attributes(lat, dm, bf);
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
    LtplVelPlan vp = {};
    vp.struct_bytes = (int32_t)sizeof(LtplVelPlan);
    vp.mode = LTPL_VP_PROFILE;
    vp.n_paths = vb->n_paths;
    vp.n_points = vb->n_points;
    vp.kappa = vb->kappa;
    vp.el = vb->el;
    vp.v_start = vb->v_start;
    vp.v_end = vb->v_end;
    vp.vx = vb->vx;
    vp.ax = vb->ax;
    vp.kappa_s = vp.el_s = vp.out_s = vb->n_points;
    return ltpl_vel_plan_batch(prm, &vp, stream);
}

int ltpl_vel_plan_batch(const LtplParams* prm, const LtplVelPlan* vp, void* stream) {
    if (!prm || !vp) return fail("null argument");
    if (vp->struct_bytes != (int32_t)sizeof(LtplVelPlan))
        return fail("vel_plan: vp.struct_bytes must be sizeof(LtplVelPlan) (the caller's layout of the struct differs)");
    const bool brake = vp->mode == LTPL_VP_BRAKE;
    if (!brake && vp->mode != LTPL_VP_PROFILE) return fail("vel_plan: vp.mode must be LTPL_VP_PROFILE or LTPL_VP_BRAKE");
    if (vp->n_paths <= 0) return fail("vel_plan: vp.n_paths must be > 0");
    const int n = vp->n_points;
    if (n < 2) return fail("vel_plan: vp.n_points must be >= 2");
    if (!vp->kappa) return fail("vel_plan: vp.kappa must be set");
    if (!vp->el) return fail("vel_plan: vp.el must be set");
    if (!vp->v_start) return fail("vel_plan: vp.v_start must be set");
    if (!brake && !vp->v_end) return fail("vel_plan: vp.v_end must be set (LTPL_VP_PROFILE)");
    if (!vp->vx) return fail("vel_plan: vp.vx must be set");
    if (!vp->ax) return fail("vel_plan: vp.ax must be set");
    if (vp->kappa_s < n) return fail("vel_plan: vp.kappa_s must be >= n_points");
    if (vp->el_s < n - 1) return fail("vel_plan: vp.el_s must be >= n_points - 1");
    if (vp->gg && vp->gg_s < 2 * (int64_t)n) return fail("vel_plan: vp.gg_s must be >= 2 n_points");
    if (vp->out_s < n) return fail("vel_plan: vp.out_s must be >= n_points");
    if (!brake) {   // the machine limits only bound the profile mode
        if (prm->n_axm < 1 || prm->n_axm > LTPL_MAX_AXM) return fail("params.n_axm out of range");
        if (prm->axm_v[prm->n_axm - 1] < prm->vel_max)
            return fail("ax_max_machines has to cover the entire velocity range of the car (i.e. >= v_max)!");
    }
    const LtplVelBatch vb = {vp->n_paths, n, vp->kappa, vp->el, vp->v_start, vp->v_end, vp->vx, vp->ax};
    VdLayout a;
    a.n_pts = vp->n_pts;
    a.gg = vp->gg;
    a.k_s = vp->kappa_s;
    a.e_s = vp->el_s;
    a.g_s = vp->gg_s;
    a.o_s = vp->out_s;
    const bool gg = vp->gg != nullptr;
    const int grid = (vp->n_paths + 31) / 32;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (brake) {
        (gg ? k_velbrake<true> : k_velbrake<false>)<<<grid, 32, vd_smem_brake(gg), st>>>(*prm, vb, a);
        return check_launch("k_velbrake");
    }
    // the dense constant-friction solver: rows of n_points and one length; anything else takes the general layout
    const bool ragged = vp->n_pts || vp->kappa_s != n || vp->el_s != n || vp->out_s != n;
    const int kind = (prm->dyn_model_exp == 1.0 ? 1 : 0) + (gg ? 2 : 0) + (ragged ? 4 : 0);
    static void (*const kFns[8])(LtplParams, LtplVelBatch, VdLayout) = {
        k_velprofile<false, false, false>, k_velprofile<true, false, false>, k_velprofile<false, true, false>,
        k_velprofile<true, true, false>,   k_velprofile<false, false, true>, k_velprofile<true, false, true>,
        k_velprofile<false, true, true>,   k_velprofile<true, true, true>};
    const int smem = (gg || ragged) ? vd_smem_general(gg) : VD_SMEM_BYTES;
    kFns[kind]<<<grid, 32, smem, st>>>(*prm, vb, a);
    return check_launch("k_velprofile");
}

static bool misaligned(const void* p, size_t a) { return ((uintptr_t)p) % a != 0; }

int ltpl_vel_follow_batch(const LtplParams* prm, const LtplVelFollow* vf, void* stream) {
    if (!prm || !vf) return fail("null argument");
    if (vf->struct_bytes != (int32_t)sizeof(LtplVelFollow))
        return fail("vel_follow: vf.struct_bytes must be sizeof(LtplVelFollow) (the caller's layout of the struct differs)");
    if (vf->n_paths <= 0) return fail("vel_follow: vf.n_paths must be > 0");
    const int n = vf->n_points;
    if (n < 2) return fail("vel_follow: vf.n_points must be >= 2");
    if (vf->n_glob < 2) return fail("vel_follow: vf.n_glob must be >= 2");
    const struct {
        const void* p;
        size_t align;
        const char* msg;
    } ptrs[] = {
        {vf->kappa, 8, "vel_follow: vf.kappa must be set and 8-byte aligned"},
        {vf->el, 8, "vel_follow: vf.el must be set and 8-byte aligned"},
        {vf->v_start, 8, "vel_follow: vf.v_start must be set and 8-byte aligned"},
        {vf->v_ego, 8, "vel_follow: vf.v_ego must be set and 8-byte aligned"},
        {vf->v_obj, 8, "vel_follow: vf.v_obj must be set and 8-byte aligned"},
        {vf->safety_d, 8, "vel_follow: vf.safety_d must be set and 8-byte aligned"},
        {vf->obj_dist, 8, "vel_follow: vf.obj_dist must be set and 8-byte aligned"},
        {vf->obj_pos, 8, "vel_follow: vf.obj_pos must be set and 8-byte aligned"},
        {vf->glob_rl, 8, "vel_follow: vf.glob_rl must be set and 8-byte aligned"},
        {vf->vx, 8, "vel_follow: vf.vx must be set and 8-byte aligned"},
        {vf->ax, 8, "vel_follow: vf.ax must be set and 8-byte aligned"},
        {vf->too_close, 1, "vel_follow: vf.too_close must be set"},
        {vf->vel_bound, 1, "vel_follow: vf.vel_bound must be set"},
    };
    for (const auto& q : ptrs)
        if (!q.p || misaligned(q.p, q.align)) return fail(q.msg);
    if (vf->n_pts && misaligned(vf->n_pts, 4)) return fail("vel_follow: vf.n_pts must be 4-byte aligned");
    if (vf->gg && misaligned(vf->gg, 8)) return fail("vel_follow: vf.gg must be 8-byte aligned");
    if (vf->kappa_s < n) return fail("vel_follow: vf.kappa_s must be >= n_points");
    if (vf->el_s < n) return fail("vel_follow: vf.el_s must be >= n_points (el has the path's n_points entries)");
    if (vf->gg && vf->gg_s < 2 * (int64_t)n) return fail("vel_follow: vf.gg_s must be >= 2 n_points");
    if (vf->obj_pos_s < 2) return fail("vel_follow: vf.obj_pos_s must be >= 2");
    if (vf->out_s < n) return fail("vel_follow: vf.out_s must be >= n_points");
    if (prm->n_axm < 1 || prm->n_axm > LTPL_MAX_AXM) return fail("params.n_axm out of range");
    if (prm->axm_v[prm->n_axm - 1] < prm->vel_max)
        return fail("ax_max_machines has to cover the entire velocity range of the car (i.e. >= v_max)!");
    if (prm->follow_control_type != 0 && prm->follow_control_type != 1)
        return fail("params.follow_control_type must be 0 (PD) or 1 (PDtan)");
    const bool gg = vf->gg != nullptr;
    const int kind = (prm->dyn_model_exp == 1.0 ? 1 : 0) + (gg ? 2 : 0);
    static void (*const kFns[4])(LtplParams, LtplVelFollow) = {k_velfollow<false, false>, k_velfollow<true, false>,
                                                               k_velfollow<false, true>, k_velfollow<true, true>};
    const int smem = vf_smem(gg);
    if (smem > 48 * 1024) {   // the attribute belongs to the kernel on the current device: raised once per device
        static std::atomic<unsigned long long> s_done{0};
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || dev >= 64) {
            (void)cudaGetLastError();
            return fail("vel_follow: no current CUDA device");
        }
        if (!(s_done.load() & (1ull << dev))) {
            std::lock_guard<std::mutex> lock(g_smem_lock);
            for (int k = 2; k < 4; ++k)
                if (cudaFuncSetAttribute((const void*)kFns[k], cudaFuncAttributeMaxDynamicSharedMemorySize, smem) !=
                    cudaSuccess) {
                    (void)cudaGetLastError();
                    return fail("k_velfollow: dynamic shared-memory attribute");
                }
            s_done.fetch_or(1ull << dev);
        }
    }
    kFns[kind]<<<(vf->n_paths + 31) / 32, 32, smem, static_cast<cudaStream_t>(stream)>>>(*prm, *vf);
    return check_launch("k_velfollow");
}

int ltpl_brake_prefix_batch(const LtplParams* prm, const LtplBrakePrefix* bp, void* stream) {
    if (!prm || !bp) return fail("null argument");
    if (bp->struct_bytes != (int32_t)sizeof(LtplBrakePrefix))
        return fail("brake_prefix: bp.struct_bytes must be sizeof(LtplBrakePrefix) (the caller's layout of the struct "
                    "differs)");
    if (bp->n_paths <= 0) return fail("brake_prefix: bp.n_paths must be > 0");
    const int n = bp->n_points;
    if (n < 2) return fail("brake_prefix: bp.n_points must be >= 2");
    if (bp->n_course_cap < 0) return fail("brake_prefix: bp.n_course_cap must be >= 0");
    const struct {
        const void* p;
        size_t align;
        const char* msg;
    } ptrs[] = {
        {bp->kappa, 8, "brake_prefix: bp.kappa must be set and 8-byte aligned"},
        {bp->el, 8, "brake_prefix: bp.el must be set and 8-byte aligned"},
        {bp->vel_plan, 8, "brake_prefix: bp.vel_plan must be set and 8-byte aligned"},
        {bp->old_gg_scale, 8, "brake_prefix: bp.old_gg_scale must be set and 8-byte aligned"},
        {bp->vx_prefix, 8, "brake_prefix: bp.vx_prefix must be set and 8-byte aligned"},
        {bp->n_prefix, 4, "brake_prefix: bp.n_prefix must be set and 4-byte aligned"},
        {bp->pref_idx, 4, "brake_prefix: bp.pref_idx must be set and 4-byte aligned"},
        {bp->vel_start, 8, "brake_prefix: bp.vel_start must be set and 8-byte aligned"},
    };
    for (const auto& q : ptrs)
        if (!q.p || misaligned(q.p, q.align)) return fail(q.msg);
    if (bp->n_course_cap > 0 && (!bp->vel_course || misaligned(bp->vel_course, 8)))
        return fail("brake_prefix: bp.vel_course must be set and 8-byte aligned (n_course_cap > 0)");
    if (bp->n_pts && misaligned(bp->n_pts, 4)) return fail("brake_prefix: bp.n_pts must be 4-byte aligned");
    if (bp->n_course && misaligned(bp->n_course, 4)) return fail("brake_prefix: bp.n_course must be 4-byte aligned");
    if (bp->gg && misaligned(bp->gg, 8)) return fail("brake_prefix: bp.gg must be 8-byte aligned");
    if (bp->kappa_s < n) return fail("brake_prefix: bp.kappa_s must be >= n_points");
    if (bp->el_s < n - 1) return fail("brake_prefix: bp.el_s must be >= n_points - 1");
    if (bp->gg && bp->gg_s < 2 * (int64_t)n) return fail("brake_prefix: bp.gg_s must be >= 2 n_points");
    if (bp->n_course_cap > 0 && bp->vel_course_s < bp->n_course_cap)
        return fail("brake_prefix: bp.vel_course_s must be >= n_course_cap");
    if (bp->vx_prefix_s < (int64_t)bp->n_course_cap + n - 1)
        return fail("brake_prefix: bp.vx_prefix_s must be >= n_course_cap + n_points - 1");
    if ((int64_t)bp->n_course_cap + n - 1 > INT32_MAX)
        return fail("brake_prefix: bp.n_course_cap + n_points - 1 must fit in int32");
    const bool gg = bp->gg != nullptr;
    (gg ? k_brakeprefix<true> : k_brakeprefix<false>)<<<(bp->n_paths + 31) / 32, 32, vd_smem_prefix(gg),
                                                         static_cast<cudaStream_t>(stream)>>>(*prm, *bp);
    return check_launch("k_brakeprefix");
}

int ltpl_path_coord_batch(const LtplPathCoord* pc, void* stream) {
    if (!pc) return fail("null argument");
    if (pc->struct_bytes != (int32_t)sizeof(LtplPathCoord))
        return fail("path_coord: pc.struct_bytes must be sizeof(LtplPathCoord) (the caller's layout of the struct "
                    "differs)");
    const int mode = pc->mode;
    if (mode < LTPL_PC_S_COORD || mode > LTPL_PC_INSIDE_BOUNDS)
        return fail("path_coord: pc.mode must be LTPL_PC_S_COORD, LTPL_PC_S_INDEX, LTPL_PC_CLOSEST or "
                    "LTPL_PC_INSIDE_BOUNDS");
    if (pc->n_queries < 0) return fail("path_coord: pc.n_queries must be >= 0");
    const int64_t m = pc->m_points;
    if (m < 2) return fail("path_coord: pc.m_points must be >= 2");
    if (pc->n_queries == 0) return 0;   // nothing is read or written
    const bool bounds = mode == LTPL_PC_INSIDE_BOUNDS;
    const struct {
        const void* p;
        size_t align;
        bool need;
        const char* msg;
    } ptrs[] = {
        {pc->x, 8, true, "path_coord: pc.x must be set and 8-byte aligned"},
        {pc->y, 8, true, "path_coord: pc.y must be set and 8-byte aligned"},
        {pc->pos, 8, true, "path_coord: pc.pos must be set and 8-byte aligned"},
        {pc->x2, 8, bounds, "path_coord: pc.x2 must be set and 8-byte aligned (LTPL_PC_INSIDE_BOUNDS)"},
        {pc->y2, 8, bounds, "path_coord: pc.y2 must be set and 8-byte aligned (LTPL_PC_INSIDE_BOUNDS)"},
        {pc->s, 8, mode == LTPL_PC_S_COORD, "path_coord: pc.s must be set (LTPL_PC_S_COORD) and 8-byte aligned"},
        {pc->closest, 4, mode <= LTPL_PC_S_INDEX,
         "path_coord: pc.closest must be set (LTPL_PC_S_COORD, LTPL_PC_S_INDEX) and 4-byte aligned"},
        {pc->idx, 4, mode == LTPL_PC_CLOSEST, "path_coord: pc.idx must be set (LTPL_PC_CLOSEST) and 4-byte aligned"},
        {pc->inside, 1, bounds, "path_coord: pc.inside must be set (LTPL_PC_INSIDE_BOUNDS)"},
        {pc->s_array, 8, false, "path_coord: pc.s_array must be 8-byte aligned"},
        {pc->n_pts, 4, false, "path_coord: pc.n_pts must be 4-byte aligned"},
    };
    for (const auto& a : ptrs)
        if ((a.need && !a.p) || (a.p && misaligned(a.p, a.align))) return fail(a.msg);
    if (pc->pt_s < 1) return fail("path_coord: pc.pt_s must be >= 1");
    if (pc->line_s != 0 && pc->line_s < (m - 1) * pc->pt_s + 1)
        return fail("path_coord: pc.line_s must be 0 (a shared line) or >= (m_points - 1) pt_s + 1");
    if (bounds && pc->pt2_s < 1) return fail("path_coord: pc.pt2_s must be >= 1");
    if (bounds && pc->line2_s != 0 && pc->line2_s < (m - 1) * pc->pt2_s + 1)
        return fail("path_coord: pc.line2_s must be 0 (a shared line) or >= (m_points - 1) pt2_s + 1");
    if (mode == LTPL_PC_S_COORD && pc->s_array) {
        if (pc->s_array_es < 1) return fail("path_coord: pc.s_array_es must be >= 1");
        if (pc->s_array_s < (m - 1) * pc->s_array_es + 1 && !(pc->s_array_s == 0 && pc->line_s == 0))
            return fail("path_coord: pc.s_array_s must be >= (m_points - 1) s_array_es + 1 (0 only with a shared line)");
    }
    if (pc->pos_s[0] < 0 || pc->pos_s[1] < 1) return fail("path_coord: pc.pos_s must be >= 0 (queries) and >= 1 (x to y)");
    using Fn = void (*)(const LtplPathCoord);
    static const Fn kFns[4] = {k_pathcoord<LTPL_PC_S_COORD>, k_pathcoord<LTPL_PC_S_INDEX>, k_pathcoord<LTPL_PC_CLOSEST>,
                               k_pathcoord<LTPL_PC_INSIDE_BOUNDS>};
    kFns[mode]<<<(unsigned)(((int64_t)pc->n_queries + PC_WARPS - 1) / PC_WARPS), PC_WARPS * 32, 0, static_cast<cudaStream_t>(stream)>>>(*pc);
    return check_launch("k_pathcoord");
}

int ltpl_stage_inputs_batch(const LtplDims* dm, const LtplBuffers* bf, const LtplStageSrc* src, void* stream) {
    if (!dm || !bf || !src) return fail("null argument");
    if (dm->batch <= 0 || dm->k_obj < 1) return fail("dims.batch and dims.k_obj must be > 0");
    if (!bf->pos || !bf->heading || !bf->vel || !bf->vel_est || !bf->n_obj || !bf->obj || !bf->zone_sel || !bf->n_pred)
        return fail("stage: buffers pos, heading, vel, vel_est, n_obj, obj, zone_sel and n_pred must be set");
    if (!src->pos || !src->heading || !src->vel || !src->n_obj || (src->k_src > 0 && !src->obj))
        return fail("stage: src.pos, src.heading, src.vel, src.n_obj and (k_src > 0) src.obj must be set");
    if (src->k_src < 0 || src->k_src > dm->k_obj) return fail("stage: src.k_src must be in [0, dims.k_obj]");
    if (src->kp_dst < 0 || (src->kp_dst > 0 && !bf->obj_pred)) return fail("stage: src.kp_dst > 0 needs buffers.obj_pred");
    if (src->pred && (!src->n_pred || src->kp_src < 0 || src->kp_src > src->kp_dst))
        return fail("stage: src.pred needs src.n_pred and src.kp_src in [0, kp_dst]");
    if (src->sel_action && (!bf->sel_action || !bf->t_const || (src->sel_action_bytes != 4 && src->sel_action_bytes != 8)))
        return fail("stage: src.sel_action needs buffers.sel_action, buffers.t_const and sel_action_bytes 4 or 8");
    if (src->restart && (!bf->restart || (src->restart_bytes != 1 && src->restart_bytes != 4 && src->restart_bytes != 8)))
        return fail("stage: src.restart needs buffers.restart and restart_bytes 1, 4 or 8");
    if (src->zone_key_rule && (!src->zone_key_last || !bf->zone_s0))
        return fail("stage: src.zone_key_rule needs src.zone_key_last and buffers.zone_s0");
    k_stage<<<ctas(dm->batch), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(*dm, *bf, *src);
    return check_launch("k_stage");
}

int ltpl_select_batch(const LtplParams* prm, const LtplDims* dm, const LtplBuffers* bf, const LtplSelect* sel,
                      void* stream) {
    if (!prm || !dm || !bf || !sel) return fail("null argument");
    if (sel->struct_bytes != (int32_t)sizeof(LtplSelect))
        return fail("select: sel.struct_bytes must be sizeof(LtplSelect) (the caller's layout of the struct differs)");
    if (dm->batch <= 0 || dm->n_export < 1) return fail("dims.batch and dims.n_export must be > 0");
    if (!bf->action_id || !bf->traj_row || !bf->traj_len || !bf->traj_id)
        return fail("select: buffers action_id, traj_row, traj_len and traj_id must be set");
    if (prm->incl_emerg_traj && !bf->em_info) return fail("select: params.incl_emerg_traj needs buffers.em_info");
    if (!sel->sel_action) return fail("select: sel.sel_action must be set");
    if (!sel->sel_info) return fail("select: sel.sel_info must be set");
    if (sel->prefer_len < 0 || sel->prefer_len > LTPL_SELECT_MAX)
        return fail("select: sel.prefer_len must be in [0, LTPL_SELECT_MAX = 8]");
    if (sel->prefer_len > 0 && !sel->prefer) return fail("select: sel.prefer must be set when sel.prefer_len > 0");
    if (sel->prefer_bytes != 1 && sel->prefer_bytes != 4 && sel->prefer_bytes != 8)
        return fail("select: sel.prefer_bytes must be 1, 4 or 8");
    if (sel->sel_traj && !bf->traj) return fail("select: sel.sel_traj needs buffers.traj");
    k_select<<<ctas(dm->batch), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(*dm, *bf, *sel, prm->incl_emerg_traj);
    return check_launch("k_select");
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
