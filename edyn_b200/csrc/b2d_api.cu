// C-ABI implementation (include/b2d.h): owns the device world, stages host SoA arrays in and out, and
// enqueues the per-step kernel sequence that stands in for stepper_sequential::update's
// bphase.update -> nphase.update -> island_manager.update -> solver.update
// (/root/reference/src/edyn/simulation/stepper_sequential.cpp:82-91).
// There is deliberately no CPU path: if CUDA is unavailable every entry point fails with B2D_ERR_CUDA.
#include "../../include/b2d.h"
#include "b2d_dist.cuh"
#include <cub/cub.cuh>
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <map>
#include <string>
#include <unordered_set>
#include <vector>
#include <chrono>
#include <unistd.h>

using namespace b2d;

static std::string g_create_error;

struct b2d_world {
    b2d_config cfg{};
    Dev d{};
    cudaStream_t stream = nullptr;
    std::vector<void *> allocs;
    std::string error;
    int num_sms = 0;
    int coop_blocks_color = 0, coop_blocks_df = 0, coop_blocks_pos_df = 0;
    int tile_fused_blocks = 0, tile_fused_blocks_2p = 0;     // grids of the island-tile kernels (CTAs loop over the tiles)
    int cell_key_bits = 48;                         // sum of d.cell_bits: end bit of the cell sort
    uint32_t bp_warp_max = 100000;                  // neighbourhood search: warp per body up to this many bodies (B2D_BP_WARP_MAX)
    bool bp_half = true;                            // thread-per-body count pass over half the neighbourhood (B2D_BP_HALF=0: the whole)
    void *cub_tmp = nullptr; size_t cub_tmp_bytes = 0;
    float *stage = nullptr; size_t stage_floats = 0;        // device staging for packed host arrays
    uint64_t launches = 0, steps = 0;
    cudaEvent_t ev_step0 = nullptr, ev_step1 = nullptr;
    // ring of per-step event pairs around the solve and integrate kernels (averaged by b2d_get_stats)
    static constexpr int RING = 256;
    cudaEvent_t ev_solve0[RING] = {}, ev_solve1[RING] = {}, ev_int0[RING] = {}, ev_int1[RING] = {};
    uint64_t timed_steps = 0;       // solver phases enqueued since the last b2d_reset_timers
    bool timed = false;
    // host mirrors needed for grid sizing / exclusions
    float max_extent = 0.0f;
    std::vector<uint32_t> large;
    std::vector<uint64_t> exclusions;
    uint32_t xhash_capacity = 0, xhash_used = 0;      // device exclusion table: slots, keys inserted (stale ones included)
    std::map<uint32_t, float2> mixing;                // material_mix_table: material_pair_key -> (friction, restitution)
    bool contacts_dirty = false;
    uint64_t updates = 0;             // island updates so far (sleep timestamps)
    // broadphase classes: bounding diameter and kind per body (host mirror), re-derived lazily before the next step
    std::vector<float> diam; std::vector<unsigned char> isdyn;
    bool class_dirty = false, ehash_dirty = true, labels_stale = true, cells_dirty = true;
    // running figures of the classification so that a hand-over (a few arrivals / departures) does not re-walk every body
    double class_sum = 0; uint64_t class_cnt = 0; float class_big = 1e30f; uint32_t class_new_first = 0; bool class_removed = false;
    std::vector<uint32_t> plan_counts;   // nranks x 4 of the current plan (bodies, manifolds, hinges, exclusions)
    // one step as CUDA graphs: [broadphase .. row preparation] [velocity solve, bracketed by the timing events]
    // [integration .. refresh].  Captured lazily, dropped whenever a host-side parameter of the sequence changes.
    bool use_graph = true, graph_valid = false;
    cudaGraphExec_t gx_pre = nullptr, gx_solve = nullptr, gx_post = nullptr, gx_all = nullptr;
    uint64_t graph_launches = 0;      // kernels one replay of the step graphs launches (a skipped island rebuild included)
    // island rebuild reuse (B2D_GRAPH_REUSE=0 turns it off): the captured step holds the rebuild under a conditional node
    // that runs it only when Counters::graph_changed is set; the body is captured on its own stream
    bool graph_reuse = true, graph_cond = false;
    cudaStream_t body_stream = nullptr;
    uint64_t host_rebuilt = 0;        // steps that ran the rebuild unconditionally (plain launches, graphs without reuse)
    bool timing = true;               // per-kernel event ring (b2d_get_stats); off = the whole step is one graph
    // multi-GPU hand-over
    std::vector<uint32_t> host_bdst;  // destination rank per body of the current plan
    uint32_t *dev_counts = nullptr;   // nranks x 4 counters of the plan
    uint32_t plan_ranks = 0;
    // raycast index (k_ray_*): allocated by the first raycast, rebuilt when state_epoch moved past ray_epoch.  Every entry
    // point that can change a body's AABB, shape or the grid parameters bumps state_epoch.
    uint64_t state_epoch = 1, ray_epoch = 0;
    RayIndex rx{};
    bool ray_alloc = false;
    void *ray_buf = nullptr; size_t ray_buf_bytes = 0;    // host-array path: rays, ignore list and results on the device
};

// Something the island rebuild reads changed behind the device kernels' back: the next step rebuilds.
static void mark_graph_changed(b2d_world *w) { cudaMemsetAsync(&w->d.cnt->graph_changed, 0x01, sizeof(uint32_t), w->stream); }
// The captured step no longer matches the world (counts, table pointers, grid pitch changed): re-capture before the next
// replay.  The executable graphs are kept so that the re-capture can patch them in place (capture()).
static void drop_graphs(b2d_world *w) { w->graph_valid = false; w->cells_dirty = true; mark_graph_changed(w); }
// B2D_TRACE=1: wall-clock marks of the hand-over entry points on stderr (development aid)
struct Trace {
    const char *what; bool on; std::chrono::steady_clock::time_point t0;
    explicit Trace(const char *w_) : what(w_), on(getenv("B2D_TRACE") != nullptr), t0(std::chrono::steady_clock::now()) {}
    void mark(const char *label) {
        if (!on) return;
        const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        fprintf(stderr, "[b2d trace pid %d] %s: %s at %.3f ms\n", (int)getpid(), what, label, ms);
    }
};
static void destroy_graphs(b2d_world *w) {
    for (cudaGraphExec_t *g : {&w->gx_pre, &w->gx_solve, &w->gx_post, &w->gx_all}) if (*g) { cudaGraphExecDestroy(*g); *g = nullptr; }
    w->graph_valid = false;
}

#define CK(call) do { cudaError_t _e = (call); if (_e != cudaSuccess) { w->error = std::string(#call) + ": " + cudaGetErrorString(_e); return B2D_ERR_CUDA; } } while (0)

template<typename T>
static bool dalloc(b2d_world *w, T *&p, size_t n, int fill = 0) {
    void *q = nullptr;
    size_t bytes = std::max<size_t>(n, 1) * sizeof(T);
    if (cudaMalloc(&q, bytes) != cudaSuccess) { w->error = "cudaMalloc failed"; return false; }
    cudaMemsetAsync(q, fill, bytes, w->stream);
    w->allocs.push_back(q);
    p = static_cast<T *>(q);
    return true;
}
// The mixing table starts with room for MIX_SLOTS / 2 entries; edits that fit are uploaded in place, so captured step
// graphs (which hold the table's pointers) stay valid.
constexpr uint32_t MIX_SLOTS = 256;
static void dfree(b2d_world *w, void *p) {
    auto it = std::find(w->allocs.begin(), w->allocs.end(), p);
    if (it != w->allocs.end()) { cudaFree(*it); w->allocs.erase(it); }
}
static uint32_t hash64_host(unsigned long long k) {      // hash64 of b2d_kernels.cuh
    k ^= k >> 33; k *= 0xff51afd7ed558ccdULL; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ULL; k ^= k >> 33;
    return (uint32_t)k;
}
static uint32_t pow2_at_least(uint64_t v) { uint32_t p = 1; while (p < v) p <<= 1; return p; }
static int blocks_for(b2d_world *w, uint64_t n, int threads) {
    uint64_t b = (n + threads - 1) / threads;
    uint64_t cap = (uint64_t)w->num_sms * 16;
    return (int)std::max<uint64_t>(1, std::min(b, cap));
}
#define LAUNCH(kernel, n, threads, ...) do { kernel<<<blocks_for(w, (n), (threads)), (threads), 0, w->stream>>>(__VA_ARGS__); ++w->launches; } while (0)

template<typename K, typename... Args>
static cudaError_t coop_launch(b2d_world *w, K kernel, int blocks, int threads, Args... args) {
    void *params[] = {(void *)&args...};
    ++w->launches;
    return cudaLaunchCooperativeKernel((void *)kernel, dim3(blocks), dim3(threads), params, 0, w->stream);
}

extern "C" {

const char *b2d_last_error(const b2d_world *w) { return w ? w->error.c_str() : g_create_error.c_str(); }

b2d_world *b2d_create(const b2d_config *cfg) {
    if (!cfg || cfg->max_bodies == 0 || cfg->max_manifolds == 0) { g_create_error = "b2d_create: bad config"; return nullptr; }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        g_create_error = "b2d_create: no CUDA device (there is no CPU fallback)"; return nullptr;
    }
    if (cudaSetDevice(cfg->device) != cudaSuccess) { g_create_error = "b2d_create: cudaSetDevice failed"; return nullptr; }
    b2d_world *w = new b2d_world();
    w->cfg = *cfg;
    if (w->cfg.fixed_dt <= 0) w->cfg.fixed_dt = 1.0f / 60.0f;
    cudaDeviceProp prop{};
    cudaGetDeviceProperties(&prop, cfg->device);
    w->num_sms = prop.multiProcessorCount;
    if (!prop.cooperativeLaunch) { g_create_error = "b2d_create: device lacks cooperative launch"; delete w; return nullptr; }
    if (cudaStreamCreateWithFlags(&w->stream, cudaStreamNonBlocking) != cudaSuccess) { g_create_error = "stream"; delete w; return nullptr; }
    cudaEventCreate(&w->ev_step0); cudaEventCreate(&w->ev_step1);

    for (int i = 0; i < b2d_world::RING; ++i) { cudaEventCreate(&w->ev_solve0[i]); cudaEventCreate(&w->ev_solve1[i]); cudaEventCreate(&w->ev_int0[i]); cudaEventCreate(&w->ev_int1[i]); }

    Dev &d = w->d;
    const uint32_t NB = cfg->max_bodies, NM = cfg->max_manifolds, NH = std::max<uint32_t>(cfg->max_hinges, 1);
    d.NB = NB; d.NM = NM; d.NH = NH; d.dt = w->cfg.fixed_dt;
    d.nbodies = 0; d.nhinges = 0; d.nlarge = 0; d.cell = 1.0f; d.inv_cell = 1.0f; d.halo_margin = HALO_MARGIN;
    for (int k = 0; k < 3; ++k) { d.cell_org[k] = -(1 << 15); d.cell_bits[k] = 16; }
    bool ok = true;
    ok = ok && dalloc(w, d.pos, NB) && dalloc(w, d.orn, NB) && dalloc(w, d.linvel, NB) && dalloc(w, d.angvel, NB);
    ok = ok && dalloc(w, d.ppos, NB) && dalloc(w, d.porn, NB);
    ok = ok && dalloc(w, d.matid, NB);
    d.mix_size = MIX_SLOTS;
    ok = ok && dalloc(w, d.mix_key, d.mix_size, 0xFF) && dalloc(w, d.mix_idx, d.mix_size) && dalloc(w, d.mix_mat, d.mix_size / 2);
    ok = ok && dalloc(w, d.dvw, 2 * (size_t)NB) && dalloc(w, d.invI, 3 * (size_t)NB) && dalloc(w, d.invIW, 3 * (size_t)NB);
    ok = ok && dalloc(w, d.grav, NB) && dalloc(w, d.shp, NB) && dalloc(w, d.bbmin, NB) && dalloc(w, d.bbmax, NB);
    ok = ok && dalloc(w, d.flags, NB) && dalloc(w, d.mat, NB) && dalloc(w, d.group, NB) && dalloc(w, d.fmask, NB);
    ok = ok && dalloc(w, d.cellkey, NB) && dalloc(w, d.cellkey_s, NB) && dalloc(w, d.cellbody, NB) && dalloc(w, d.cellbody_s, NB) && dalloc(w, d.brank, NB);
    ok = ok && dalloc(w, d.bprec_min, NB) && dalloc(w, d.bprec_max, NB) && dalloc(w, d.cell_box, 6);
    d.chash_size = pow2_at_least(2ull * NB);
    ok = ok && dalloc(w, d.chash_key, d.chash_size, 0xFF) && dalloc(w, d.chash_val, d.chash_size);
    // direct cell table: DENSE_CELLS_PER_BODY cells per body; B2D_BP_CELL_TABLE overrides the factor (0: the cell hash on every step)
    uint64_t cells_per_body = DENSE_CELLS_PER_BODY;
    if (const char *e = getenv("B2D_BP_CELL_TABLE")) cells_per_body = (uint64_t)std::max(0, atoi(e));
    d.cstart_size = (uint32_t)std::min<uint64_t>(cells_per_body * NB, 0xFFFFFFFFull);
    ok = ok && dalloc(w, d.cstart, d.cstart_size, 0xFF);
    if (const char *e = getenv("B2D_BP_HALF")) w->bp_half = atoi(e) != 0;
    ok = ok && dalloc(w, d.large_list, NB) && dalloc(w, d.lmask, NB) && dalloc(w, d.newcount, NB) && dalloc(w, d.newoff, NB) && dalloc(w, d.newpairs, NM);
    ok = ok && dalloc(w, d.free_flag, NM) && dalloc(w, d.free_rank, NM) && dalloc(w, d.free_list, NM);
    d.mhash_size = pow2_at_least(2ull * NM);
    ok = ok && dalloc(w, d.mhash_key, d.mhash_size, 0xFF) && dalloc(w, d.mhash_val, d.mhash_size);
    d.xhash_size = 0; d.xhash_key = nullptr;
    ok = ok && dalloc(w, d.mpair, NM) && dalloc(w, d.mstate, NM);
    ok = ok && dalloc(w, d.pA, 4 * (size_t)NM) && dalloc(w, d.pB, 4 * (size_t)NM) && dalloc(w, d.pN, 4 * (size_t)NM);
    ok = ok && dalloc(w, d.pL, 4 * (size_t)NM) && dalloc(w, d.pI, 4 * (size_t)NM) && dalloc(w, d.clist, NM);
    ok = ok && dalloc(w, d.parent, NB) && dalloc(w, d.bmask, NB) && dalloc(w, d.jmask, NB) && dalloc(w, d.prop, NB) && dalloc(w, d.jprop, NB);
    ok = ok && dalloc(w, d.ckey, NM) && dalloc(w, d.ckey_s, NM) && dalloc(w, d.cidx, NM) && dalloc(w, d.cidx_s, NM) && dalloc(w, d.npidx, NM);
    ok = ok && dalloc(w, d.hkey, NH) && dalloc(w, d.hkey_s, NH) && dalloc(w, d.hidx, NH) && dalloc(w, d.hidx_s, NH);
    // island tiles: the census arrays are one allocation (zeroed together every step), so are the per-tile tables
    d.max_tiles = (uint32_t)std::min<uint64_t>(((uint64_t)NB + NM + NH) / TILE_ISLAND_MAX + 64, 1u << KEY_TILE_BITS);   // beyond: dataflow path
    ok = ok && dalloc(w, d.isl_nb, 3 * (size_t)NB) && dalloc(w, d.swgt, NB) && dalloc(w, d.swsum, NB) && dalloc(w, d.btile, NB, 0xFF) && dalloc(w, d.bslot, NB, 0xFF);
    d.isl_nm = d.isl_nb + NB; d.isl_nh = d.isl_nb + 2 * (size_t)NB;
    ok = ok && dalloc(w, d.tile_nb, 5 * (size_t)d.max_tiles) && dalloc(w, d.tile_body, (size_t)d.max_tiles * TILE_CAP);
    d.tile_c0 = d.tile_nb + d.max_tiles; d.tile_c1 = d.tile_c0 + d.max_tiles; d.tile_h0 = d.tile_c1 + d.max_tiles; d.tile_h1 = d.tile_h0 + d.max_tiles;
    ok = ok && dalloc(w, d.tile_hdr, d.max_tiles) && dalloc(w, d.tplan_h, (size_t)d.max_tiles * TILE_CAP) && dalloc(w, d.tplan_c, (size_t)d.max_tiles * TILE_CAP);
    ok = ok && dalloc(w, d.tplan_w, (size_t)d.max_tiles * TILE_CAP);
    ok = ok && dalloc(w, d.isl_err, NB) && dalloc(w, d.isl_done, NB);
    ok = ok && dalloc(w, d.hdr, NM) && dalloc(w, d.R0, 4 * (size_t)NM) && dalloc(w, d.R1, 4 * (size_t)NM) && dalloc(w, d.R2, 4 * (size_t)NM);
    ok = ok && dalloc(w, d.R3, 4 * (size_t)NM) && dalloc(w, d.IMP, 4 * (size_t)NM);
    ok = ok && dalloc(w, d.hpair, NH) && dalloc(w, d.hpivA, NH) && dalloc(w, d.hpivB, NH) && dalloc(w, d.hfA0, NH) && dalloc(w, d.hfA1, NH);
    ok = ok && dalloc(w, d.hfA2, NH) && dalloc(w, d.hfB0, NH) && dalloc(w, d.himp, 5 * (size_t)NH) && dalloc(w, d.hcolor, NH, 0xFF);
    ok = ok && dalloc(w, d.HR, 7 * (size_t)NH) && dalloc(w, d.hhdr, NH) && dalloc(w, d.cnt, 1);
    ok = ok && dalloc(w, d.tkt, NM) && dalloc(w, d.htkt, NH) && dalloc(w, d.pisl, NM) && dalloc(w, d.hisl, NH) && dalloc(w, d.prec, 3 * NB);
    d.ehash_size = pow2_at_least(2ull * NB);
    ok = ok && dalloc(w, d.entity, NB) && dalloc(w, d.ehash, d.ehash_size, 0xFF) && dalloc(w, d.ibox, 6 * (size_t)NB) && dalloc(w, d.isl_dst, NB, 0xFF) && dalloc(w, d.bdst, NB, 0xFF);
    ok = ok && dalloc(w, w->dev_counts, 4 * 64);
    if (cfg->flags & B2D_FLAG_RESTITUTION_SOLVER) {
        d.rest_iters = 8; d.rest_individual = 3;                  // context/settings.hpp:29-30
        ok = ok && dalloc(w, d.rcnt, NB) && dalloc(w, d.roff, NB) && dalloc(w, d.rcur, NB) && dalloc(w, d.rstamp, NB) && dalloc(w, d.rnext, NB)
                && dalloc(w, d.radj, 2 * ((size_t)NM + NH)) && dalloc(w, d.radj_m, 2 * ((size_t)NM + NH));
    }
    d.sleeping = (cfg->flags & B2D_FLAG_SLEEPING) ? 1u : 0u;
    if (d.sleeping) {
        ok = ok && dalloc(w, d.prev_label, NB, 0xFF) && dalloc(w, d.isl_size, NB) && dalloc(w, d.size_new, NB) && dalloc(w, d.isl_flags, NB)
                && dalloc(w, d.contributor, NB) && dalloc(w, d.heir, NB) && dalloc(w, d.isl_ts, NB) && dalloc(w, d.ts_new, NB);
    }
    // hcolor must hold COLOR_NONE (0xFF as a 32-bit value), not 0xFFFFFFFF
    if (ok) { std::vector<uint32_t> hc(NH, COLOR_NONE); cudaMemcpyAsync(d.hcolor, hc.data(), NH * sizeof(uint32_t), cudaMemcpyHostToDevice, w->stream); cudaStreamSynchronize(w->stream); }

    // CUB temp storage: the largest of the sorts/scans used per step
    size_t need = 0, t = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, t, d.cellkey, d.cellkey_s, d.cellbody, d.cellbody_s, (int)NB, 0, 48, w->stream); need = std::max(need, t);
    cub::DeviceRadixSort::SortPairs(nullptr, t, d.ckey, d.ckey_s, d.cidx, d.cidx_s, (int)NM, 0, COLOR_KEY_BITS, w->stream); need = std::max(need, t);
    cub::DeviceScan::ExclusiveSum(nullptr, t, d.free_flag, d.free_rank, (int)NM, w->stream); need = std::max(need, t);
    cub::DeviceScan::ExclusiveSum(nullptr, t, d.newcount, d.newoff, (int)NB, w->stream); need = std::max(need, t);
    cub::DeviceRadixSort::SortPairs(nullptr, t, d.hkey, d.hkey_s, d.hidx, d.hidx_s, (int)NH, 0, COLOR_KEY_BITS, w->stream); need = std::max(need, t);
    cub::DeviceScan::ExclusiveSum(nullptr, t, d.swgt, d.swsum, (int)NB, w->stream); need = std::max(need, t);
    cub::DeviceScan::ExclusiveSum(nullptr, t, d.hidx, d.hidx_s, (int)NH, w->stream); need = std::max(need, t);
    w->cub_tmp_bytes = need + 256;
    void *tmp = nullptr;
    if (ok && cudaMalloc(&tmp, w->cub_tmp_bytes) != cudaSuccess) ok = false;
    w->cub_tmp = tmp; if (tmp) w->allocs.push_back(tmp);
    w->stage_floats = (size_t)NB * 32 + (size_t)NM * 80;
    float *st = nullptr;
    if (ok && cudaMalloc(&st, w->stage_floats * sizeof(float)) != cudaSuccess) ok = false;
    w->stage = st; if (st) w->allocs.push_back(st);

    // Persistent kernels: co-resident grids.  The colouring kernel has a grid barrier per round (its cost grows with the
    // CTA count): a few CTAs per SM.  The dataflow solve wants every resident warp it can get (latency hiding, no
    // barrier cost per CTA).  The island-tile kernels need no co-residency: their CTAs loop over the tiles.
    int per_sm = 0, want = 2;
    if (const char *e = getenv("B2D_COOP_BLOCKS_PER_SM")) want = std::max(1, atoi(e));
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_color, 256, 0); w->coop_blocks_color = std::max(1, std::min(per_sm, want)) * w->num_sms;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_solve_df, B2D_SOLVE_THREADS, 0); w->coop_blocks_df = std::max(1, per_sm) * w->num_sms;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_position_df, B2D_POS_THREADS, 0); w->coop_blocks_pos_df = std::max(1, per_sm) * w->num_sms;
    cudaFuncSetAttribute(k_island_tiles, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TILE_FUSED_SMEM);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_island_tiles, TILE_CAP, TILE_FUSED_SMEM); w->tile_fused_blocks = std::max(1, per_sm) * w->num_sms;
    cudaFuncSetAttribute(k_island_tiles_2p, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TILE_FUSED_SMEM_2P);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_island_tiles_2p, TILE_CAP, TILE_FUSED_SMEM_2P); w->tile_fused_blocks_2p = std::max(1, per_sm) * w->num_sms;
    if (const char *e = getenv("B2D_BP_WARP_MAX")) w->bp_warp_max = (uint32_t)std::max(0, atoi(e));
    if (const char *e = getenv("B2D_TILES")) if (atoi(e) == 0) d.max_tiles = 0;          // development: everything through the dataflow path
    if (const char *e = getenv("B2D_GRAPH")) w->use_graph = atoi(e) != 0;
    if (const char *e = getenv("B2D_GRAPH_REUSE")) w->graph_reuse = atoi(e) != 0;     // 0: graphs rebuild the islands every step
    if (w->use_graph && w->graph_reuse && cudaStreamCreateWithFlags(&w->body_stream, cudaStreamNonBlocking) != cudaSuccess) { cudaGetLastError(); w->body_stream = nullptr; w->graph_reuse = false; }

    if (!ok || cudaStreamSynchronize(w->stream) != cudaSuccess) {
        g_create_error = "b2d_create: device allocation failed: " + w->error;
        b2d_destroy(w);
        return nullptr;
    }
    return w;
}

void b2d_destroy(b2d_world *w) {
    if (!w) return;
    cudaSetDevice(w->cfg.device);
    if (w->stream) cudaStreamSynchronize(w->stream);
    destroy_graphs(w);
    for (void *p : w->allocs) cudaFree(p);
    if (w->ray_buf) cudaFree(w->ray_buf);
    if (w->ev_step0) cudaEventDestroy(w->ev_step0);
    if (w->ev_step1) cudaEventDestroy(w->ev_step1);
    for (int i = 0; i < b2d_world::RING; ++i) for (cudaEvent_t e : {w->ev_solve0[i], w->ev_solve1[i], w->ev_int0[i], w->ev_int1[i]}) if (e) cudaEventDestroy(e);
    if (w->body_stream) cudaStreamDestroy(w->body_stream);
    if (w->stream) cudaStreamDestroy(w->stream);
    delete w;
}

void *b2d_stream(b2d_world *w) { return w ? (void *)w->stream : nullptr; }
// Device-side overflow flags become return codes here (the step itself is asynchronous).
static int check_device_flags(b2d_world *w) {
    uint32_t err = 0;
    CK(cudaMemcpyAsync(&err, &w->d.cnt->err, sizeof(uint32_t), cudaMemcpyDeviceToHost, w->stream));
    CK(cudaStreamSynchronize(w->stream));
    if (!err) return B2D_OK;
    w->error = "device error flags:";
    if (err & ERR_MANIFOLD_CAPACITY) w->error += " max_manifolds exceeded;";
    if (err & ERR_LARGE_CAPACITY) w->error += " large-body list overflow;";
    if (err & ERR_COLOR_OVERFLOW) w->error += " a contact or joint found all 64 colours taken on its dynamic bodies together;";
    if (err & ERR_SOLVER_TIMEOUT) w->error += " solver dataflow wait timed out;";
    if (err & ERR_RESTITUTION_GROUP) w->error += " restitution solver: more than 32 closing manifolds or 96 contact points at one body;";
    if (err & ERR_UNKNOWN_ENTITY) w->error += " hand-over blob names an unknown entity;";
    if (err & (ERR_MANIFOLD_CAPACITY | ERR_LARGE_CAPACITY)) return B2D_ERR_CAPACITY;
    if (err & (ERR_COLOR_OVERFLOW | ERR_RESTITUTION_GROUP)) return B2D_ERR_UNSUPPORTED;
    return B2D_ERR_CUDA;
}
int b2d_sync(b2d_world *w) { if (!w) return B2D_ERR_ARGUMENT; cudaSetDevice(w->cfg.device); CK(cudaStreamSynchronize(w->stream)); return check_device_flags(w); }

// Bounding diameter of a shape: an upper bound of any AABB extent it can have.
static float shape_diameter(uint32_t kind, const float *p) {
    switch (kind) {
    case B2D_SHAPE_SPHERE: return 2 * p[0];
    case B2D_SHAPE_CAPSULE: return 2 * (p[0] + p[1]);
    case B2D_SHAPE_BOX: return 2 * std::sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]);
    default: return INFINITY;
    }
}

// Broadphase classes, world-wide: the grid pitch is the largest bounding diameter among the bodies that go into the
// grid; planes and bodies much larger than the typical dynamic body (4 x the mean dynamic diameter of the WHOLE world,
// however the bodies were batched) are kept in a brute-force list instead.  Runs before the first step after the body
// population changed; results do not depend on the classification (the exact AABB tests decide), only speed does.  A
// large DYNAMIC body also searches brute force, and its constraints are filed under it, or under its small dynamic
// partner (key_body): tests/test_gpu_large_bodies.py holds both to the oracle.
static void class_add(b2d_world *w, float diam, bool dyn) {
    w->diam.push_back(diam); w->isdyn.push_back(dyn ? 1 : 0);
    if (dyn && diam > 0 && std::isfinite(diam)) { w->class_sum += diam; ++w->class_cnt; }
}
static void class_forget(b2d_world *w, uint32_t i) {
    if (w->isdyn[i] && w->diam[i] > 0 && std::isfinite(w->diam[i])) { w->class_sum -= w->diam[i]; --w->class_cnt; }
    w->diam[i] = 0.0f; w->isdyn[i] = 0;
}
static int reclassify(b2d_world *w) {
    Dev &d = w->d;
    double sum = 0; uint64_t cnt = 0;
    for (uint32_t i = 0; i < d.nbodies; ++i) if (w->isdyn[i] && w->diam[i] > 0 && std::isfinite(w->diam[i])) { sum += w->diam[i]; ++cnt; }
    const float big = cnt ? float(4.0 * sum / cnt) : 1e30f;
    w->class_sum = sum; w->class_cnt = cnt; w->class_big = big; w->class_new_first = d.nbodies; w->class_removed = false;
    w->large.clear(); w->max_extent = 0.0f;
    for (uint32_t i = 0; i < d.nbodies; ++i) {
        const float dm = w->diam[i];
        if (dm <= 0) continue;                                       // shapeless or removed
        if (!std::isfinite(dm) || dm > big) w->large.push_back(i);
        else w->max_extent = std::max(w->max_extent, dm);
    }
    cudaStream_t s = w->stream;
    if (!w->large.empty()) CK(cudaMemcpyAsync(d.large_list, w->large.data(), w->large.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
    d.nlarge = (uint32_t)w->large.size();
    d.cell = w->max_extent + 2 * BREAKING_THRESHOLD + 1e-3f;
    d.inv_cell = 1.0f / d.cell;
    if (d.nbodies) { LAUNCH(k_large_clear, d.nbodies, 256, d); if (d.nlarge) LAUNCH(k_large_set, d.nlarge, 256, d); }
    CK(cudaStreamSynchronize(s));
    w->class_dirty = false;
    drop_graphs(w);
    return B2D_OK;
}

int b2d_add_bodies(b2d_world *w, const b2d_bodies *b, uint32_t *first_id) {
    if (!w || !b) return B2D_ERR_ARGUMENT;
    cudaSetDevice(w->cfg.device);
    ++w->state_epoch;
    Dev &d = w->d;
    const uint32_t n = b->count, first = d.nbodies;
    if (first + (uint64_t)n > d.NB) { w->error = "b2d_add_bodies: max_bodies exceeded"; return B2D_ERR_CAPACITY; }
    for (uint32_t i = 0; i < n; ++i) {
        uint32_t sk = b->shape_kind[i];
        if (!(sk == B2D_SHAPE_SPHERE || sk == B2D_SHAPE_CAPSULE || sk == B2D_SHAPE_BOX || sk == B2D_SHAPE_PLANE || sk == B2D_SHAPE_NONE)) {
            w->error = "b2d_add_bodies: shape kind outside the hot-path scope (sphere, capsule, box, plane)"; return B2D_ERR_UNSUPPORTED;
        }
        if (sk == B2D_SHAPE_PLANE && b->kind[i] != B2D_STATIC) { w->error = "b2d_add_bodies: plane shapes must be static"; return B2D_ERR_UNSUPPORTED; }
        if (b->kind[i] > B2D_STATIC) { w->error = "b2d_add_bodies: bad body kind"; return B2D_ERR_ARGUMENT; }
        if (b->material && b->material[i] > B2D_MATERIAL_UNASSIGNED && b->material[i] != B2D_MATERIAL_NONE) {
            w->error = "b2d_add_bodies: material must be an id up to 0xFFFF or B2D_MATERIAL_NONE"; return B2D_ERR_ARGUMENT;
        }
    }
    std::vector<float4> pos(n), orn(n), lv(n), av(n), invI(3 * (size_t)n), grav(n), shp(n);
    std::vector<uint32_t> flags(n), matid(n); std::vector<float2> mat(n); std::vector<unsigned long long> grp(n), msk(n);
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t kind = b->kind[i], sk = b->shape_kind[i];
        const bool dyn = kind == B2D_DYNAMIC;
        pos[i] = make_float4(b->pos[3 * i], b->pos[3 * i + 1], b->pos[3 * i + 2], dyn ? b->inv_mass[i] : 0.0f);
        orn[i] = make_float4(b->orn[4 * i], b->orn[4 * i + 1], b->orn[4 * i + 2], b->orn[4 * i + 3]);
        if (kind == B2D_STATIC) { lv[i] = av[i] = make_float4(0, 0, 0, 0); }
        else { lv[i] = make_float4(b->linvel[3 * i], b->linvel[3 * i + 1], b->linvel[3 * i + 2], 0); av[i] = make_float4(b->angvel[3 * i], b->angvel[3 * i + 1], b->angvel[3 * i + 2], 0); }
        for (int r = 0; r < 3; ++r) invI[3 * (size_t)i + r] = dyn ? make_float4(b->inv_inertia[9 * i + 3 * r], b->inv_inertia[9 * i + 3 * r + 1], b->inv_inertia[9 * i + 3 * r + 2], 0) : make_float4(0, 0, 0, 0);
        grav[i] = make_float4(b->gravity[3 * i], b->gravity[3 * i + 1], b->gravity[3 * i + 2], 0);
        shp[i] = make_float4(b->shape_params[4 * i], b->shape_params[4 * i + 1], b->shape_params[4 * i + 2], b->shape_params[4 * i + 3]);
        uint32_t f = kind | (sk << F_SHAPE_SHIFT);
        if (dyn && (sk == B2D_SHAPE_SPHERE || sk == B2D_SHAPE_CAPSULE)) f |= F_ROLLING;
        unsigned long long g = b->group ? b->group[i] : ~0ULL, m = b->mask ? b->mask[i] : ~0ULL;
        if (b->group && b->mask && !(g == ~0ULL && m == ~0ULL)) f |= F_FILTER;
        const uint32_t mid = b->material ? b->material[i] : B2D_MATERIAL_UNASSIGNED;
        if (mid == B2D_MATERIAL_NONE) f |= F_SENSOR;
        if (b->presentation && b->presentation[i]) f |= F_PRESENT;
        matid[i] = mid == B2D_MATERIAL_NONE ? MATERIAL_UNASSIGNED : mid;
        class_add(w, sk != B2D_SHAPE_NONE ? shape_diameter(sk, b->shape_params + 4 * i) : 0.0f, dyn);
        flags[i] = f; mat[i] = make_float2(b->friction[i], b->restitution[i]); grp[i] = g; msk[i] = m;
    }
    cudaStream_t s = w->stream;
    CK(cudaMemcpyAsync(d.pos + first, pos.data(), n * sizeof(float4), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d.orn + first, orn.data(), n * sizeof(float4), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d.ppos + first, pos.data(), n * sizeof(float4), cudaMemcpyHostToDevice, s));     // make_rigidbody: def.position
    CK(cudaMemcpyAsync(d.porn + first, orn.data(), n * sizeof(float4), cudaMemcpyHostToDevice, s));     // and def.orientation
    CK(cudaMemcpyAsync(d.linvel + first, lv.data(), n * sizeof(float4), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d.angvel + first, av.data(), n * sizeof(float4), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d.invI + 3 * (size_t)first, invI.data(), 3 * (size_t)n * sizeof(float4), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d.grav + first, grav.data(), n * sizeof(float4), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d.shp + first, shp.data(), n * sizeof(float4), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d.flags + first, flags.data(), n * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d.mat + first, mat.data(), n * sizeof(float2), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d.matid + first, matid.data(), n * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d.group + first, grp.data(), n * sizeof(unsigned long long), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d.fmask + first, msk.data(), n * sizeof(unsigned long long), cudaMemcpyHostToDevice, s));
    d.nbodies = first + n;
    LAUNCH(k_entities_default, n, 256, d, first, n);
    LAUNCH(k_refresh_bodies, n, 256, d, first, n);
    CK(cudaStreamSynchronize(s));
    w->class_dirty = true;
    drop_graphs(w);
    if (first_id) *first_id = first;
    return B2D_OK;
}

int b2d_remove_bodies(b2d_world *w, const uint32_t *ids, uint32_t n) {
    if (!w || (n && !ids)) return B2D_ERR_ARGUMENT;
    cudaSetDevice(w->cfg.device);
    ++w->state_epoch;
    Dev &d = w->d;
    for (uint32_t k = 0; k < n; ++k) if (ids[k] >= d.nbodies) { w->error = "b2d_remove_bodies: body id out of range"; return B2D_ERR_ARGUMENT; }
    if (!n) return B2D_OK;
    cudaStream_t s = w->stream;
    if ((size_t)n > w->stage_floats) { w->error = "b2d_remove_bodies: more ids than the staging buffer holds"; return B2D_ERR_CAPACITY; }
    uint32_t *dev_ids = (uint32_t *)w->stage;          // the staging buffer doubles as scratch: every user synchronises before it returns
    CK(cudaMemcpyAsync(dev_ids, ids, n * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
    LAUNCH(k_remove_bodies, n, 256, d, dev_ids, n);
    if (d.nhinges) LAUNCH(k_remove_hinges, d.nhinges, 256, d);
    // destroying a node queues its island for wake-up (island_manager.cpp:74-97); restated coarsely: everybody wakes
    if (d.sleeping) LAUNCH(k_wake_bodies, d.nbodies, 256, d, (const uint32_t *)nullptr, d.nbodies);
    CK(cudaStreamSynchronize(s));
    for (uint32_t k = 0; k < n; ++k) class_forget(w, ids[k]);
    w->contacts_dirty = true; w->class_dirty = true; w->ehash_dirty = true;
    drop_graphs(w);
    return B2D_OK;
}

int b2d_wake_bodies(b2d_world *w, const uint32_t *ids, uint32_t n) {
    if (!w) return B2D_ERR_ARGUMENT;
    cudaSetDevice(w->cfg.device);
    Dev &d = w->d;
    cudaStream_t s = w->stream;
    mark_graph_changed(w);                              // sleeping flags decide which constraints have rows
    if (!ids) { if (d.nbodies) LAUNCH(k_wake_bodies, d.nbodies, 256, d, (const uint32_t *)nullptr, d.nbodies); CK(cudaStreamSynchronize(s)); return B2D_OK; }
    for (uint32_t k = 0; k < n; ++k) if (ids[k] >= d.nbodies) { w->error = "b2d_wake_bodies: body id out of range"; return B2D_ERR_ARGUMENT; }
    if (!n) return B2D_OK;
    if ((size_t)n > w->stage_floats) { w->error = "b2d_wake_bodies: more ids than the staging buffer holds"; return B2D_ERR_CAPACITY; }
    uint32_t *dev_ids = (uint32_t *)w->stage;
    CK(cudaMemcpyAsync(dev_ids, ids, n * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
    LAUNCH(k_wake_bodies, n, 256, d, (const uint32_t *)dev_ids, n);
    CK(cudaStreamSynchronize(s));
    return B2D_OK;
}

int b2d_download_sleeping(b2d_world *w, uint32_t *asleep) {
    if (!w || !asleep) return B2D_ERR_ARGUMENT;
    cudaSetDevice(w->cfg.device);
    Dev &d = w->d;
    CK(cudaMemcpyAsync(asleep, d.flags, d.nbodies * sizeof(uint32_t), cudaMemcpyDeviceToHost, w->stream));
    CK(cudaStreamSynchronize(w->stream));
    for (uint32_t i = 0; i < d.nbodies; ++i) asleep[i] = (asleep[i] & F_SLEEPING) ? 1u : 0u;
    return B2D_OK;
}

static void plane_space_host(const float *n, float *p, float *q) {   // geom.cpp:730-754
    if (std::fabs(n[2]) > 0.7071067811865475244f) {
        float a = n[1] * n[1] + n[2] * n[2]; float k = 1.0f / std::sqrt(a);
        p[0] = 0; p[1] = -n[2] * k; p[2] = n[1] * k; q[0] = a * k; q[1] = -n[0] * p[2]; q[2] = n[0] * p[1];
    } else {
        float a = n[0] * n[0] + n[1] * n[1]; float k = 1.0f / std::sqrt(a);
        p[0] = -n[1] * k; p[1] = n[0] * k; p[2] = 0; q[0] = -n[2] * p[1]; q[1] = n[2] * p[0]; q[2] = a * k;
    }
}

int b2d_add_hinges(b2d_world *w, uint32_t n, const uint32_t *a, const uint32_t *b, const float *pivA, const float *pivB,
                   const float *axA, const float *axB) {
    if (!w) return B2D_ERR_ARGUMENT;
    cudaSetDevice(w->cfg.device);
    Dev &d = w->d;
    const uint32_t first = d.nhinges;
    if (first + (uint64_t)n > w->cfg.max_hinges) { w->error = "b2d_add_hinges: max_hinges exceeded"; return B2D_ERR_CAPACITY; }
    std::vector<uint2> pr(n); std::vector<float4> pa(n), pb(n), f0(n), f1(n), f2(n), g0(n);
    for (uint32_t i = 0; i < n; ++i) {
        if (a[i] >= d.nbodies || b[i] >= d.nbodies) { w->error = "b2d_add_hinges: body id out of range"; return B2D_ERR_ARGUMENT; }
        pr[i] = make_uint2(a[i], b[i]);
        pa[i] = make_float4(pivA[3 * i], pivA[3 * i + 1], pivA[3 * i + 2], 0); pb[i] = make_float4(pivB[3 * i], pivB[3 * i + 1], pivB[3 * i + 2], 0);
        float p[3], q[3];
        plane_space_host(axA + 3 * i, p, q);       // set_axes, hinge_constraint.cpp:11-17
        f0[i] = make_float4(axA[3 * i], axA[3 * i + 1], axA[3 * i + 2], 0); f1[i] = make_float4(p[0], p[1], p[2], 0); f2[i] = make_float4(q[0], q[1], q[2], 0);
        g0[i] = make_float4(axB[3 * i], axB[3 * i + 1], axB[3 * i + 2], 0);
    }
    cudaStream_t s = w->stream;
    CK(cudaMemcpyAsync(d.hpair + first, pr.data(), n * sizeof(uint2), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d.hpivA + first, pa.data(), n * sizeof(float4), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d.hpivB + first, pb.data(), n * sizeof(float4), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d.hfA0 + first, f0.data(), n * sizeof(float4), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d.hfA1 + first, f1.data(), n * sizeof(float4), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d.hfA2 + first, f2.data(), n * sizeof(float4), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d.hfB0 + first, g0.data(), n * sizeof(float4), cudaMemcpyHostToDevice, s));
    CK(cudaMemsetAsync(d.himp + 5 * (size_t)first, 0, 5 * (size_t)n * sizeof(float), s));
    CK(cudaStreamSynchronize(s));
    d.nhinges = first + n;
    drop_graphs(w);
    return B2D_OK;
}

// collision_exclusion as a pair hash set, rebuilt on every change (host list -> device open-addressing table)
static int upload_exclusions(b2d_world *w) {
    Dev &d = w->d;
    uint32_t size = pow2_at_least(4ull * w->exclusions.size() + 1024);    // load <= 1/4: room for insert_exclusions
    std::vector<unsigned long long> table(size, ~0ULL);
    for (uint64_t k : w->exclusions) {
        uint32_t h = hash64_host(k) & (size - 1);
        while (table[h] != ~0ULL && table[h] != k) h = (h + 1) & (size - 1);
        table[h] = k;
    }
    unsigned long long *dev = nullptr;
    if (!dalloc(w, dev, size)) return B2D_ERR_CUDA;
    CK(cudaMemcpyAsync(dev, table.data(), size * sizeof(unsigned long long), cudaMemcpyHostToDevice, w->stream));
    CK(cudaStreamSynchronize(w->stream));
    if (d.xhash_key) dfree(w, d.xhash_key);             // the table this one replaces
    d.xhash_key = dev; d.xhash_size = w->exclusions.empty() ? 0u : size;
    w->xhash_capacity = size; w->xhash_used = (uint32_t)w->exclusions.size();
    drop_graphs(w);
    return B2D_OK;
}
// Append pairs that are known to be new (the ids of arriving bodies are fresh) without rebuilding the table: entries of
// departed bodies stay behind as harmless garbage (ids are never reused) until the load factor asks for a rebuild.
static int insert_exclusions(b2d_world *w, const std::vector<uint64_t> &keys) {
    if (keys.empty()) return B2D_OK;
    Dev &d = w->d;
    w->exclusions.insert(w->exclusions.end(), keys.begin(), keys.end());
    if (!d.xhash_key || d.xhash_size == 0 || 2ull * (w->xhash_used + keys.size()) > w->xhash_capacity) return upload_exclusions(w);
    if (keys.size() * 2 > w->stage_floats) return upload_exclusions(w);
    unsigned long long *tmp = (unsigned long long *)w->stage;
    CK(cudaMemcpyAsync(tmp, keys.data(), keys.size() * sizeof(uint64_t), cudaMemcpyHostToDevice, w->stream));
    LAUNCH(k_xhash_insert, keys.size(), 256, d, (const unsigned long long *)tmp, (uint32_t)keys.size());
    mark_graph_changed(w);
    CK(cudaStreamSynchronize(w->stream));             // `keys` may go out of scope, the staging buffer be reused
    w->xhash_used += (uint32_t)keys.size();
    return B2D_OK;
}

int b2d_add_exclusions(b2d_world *w, uint32_t n, const uint32_t *a, const uint32_t *b) {
    if (!w || (n && (!a || !b))) return B2D_ERR_ARGUMENT;
    cudaSetDevice(w->cfg.device);
    std::unordered_set<uint64_t> seen(w->exclusions.begin(), w->exclusions.end());
    for (uint32_t i = 0; i < n; ++i) {
        if (a[i] >= w->d.nbodies || b[i] >= w->d.nbodies) { w->error = "b2d_add_exclusions: body id out of range"; return B2D_ERR_ARGUMENT; }
        uint64_t lo = std::min(a[i], b[i]), hi = std::max(a[i], b[i]);
        const uint64_t k = (lo << 32) | hi;
        if (seen.insert(k).second) w->exclusions.push_back(k);
    }
    return upload_exclusions(w);
}

int b2d_remove_exclusions(b2d_world *w, uint32_t n, const uint32_t *a, const uint32_t *b) {
    if (!w || (n && (!a || !b))) return B2D_ERR_ARGUMENT;
    cudaSetDevice(w->cfg.device);
    std::unordered_set<uint64_t> gone;
    for (uint32_t i = 0; i < n; ++i) {
        uint64_t lo = std::min(a[i], b[i]), hi = std::max(a[i], b[i]);
        gone.insert((lo << 32) | hi);
    }
    w->exclusions.erase(std::remove_if(w->exclusions.begin(), w->exclusions.end(), [&](uint64_t k) { return gone.count(k) != 0; }), w->exclusions.end());
    return upload_exclusions(w);
}

// material_mix_table on the device: the whole table is re-hashed on the host and uploaded in place; only when it outgrows
// its slots is it reallocated, which invalidates the captured step graphs.
static int upload_mixing(b2d_world *w) {
    Dev &d = w->d;
    uint32_t size = d.mix_size;
    while (2ull * w->mixing.size() > size) size *= 2;
    std::vector<unsigned long long> keys(size, EMPTY_KEY);
    std::vector<uint32_t> idx(size, 0);
    std::vector<float2> mat(size / 2);
    uint32_t k = 0;
    for (const auto &e : w->mixing) {
        uint32_t h = hash64_host(e.first) & (size - 1);
        while (keys[h] != EMPTY_KEY) h = (h + 1) & (size - 1);
        keys[h] = e.first; idx[h] = k; mat[k++] = e.second;
    }
    if (size != d.mix_size) {
        CK(cudaStreamSynchronize(w->stream));
        dfree(w, d.mix_key); dfree(w, d.mix_idx); dfree(w, d.mix_mat);
        if (!dalloc(w, d.mix_key, size) || !dalloc(w, d.mix_idx, size) || !dalloc(w, d.mix_mat, size / 2)) return B2D_ERR_CUDA;
        d.mix_size = size;
        drop_graphs(w);
    }
    CK(cudaMemcpyAsync(d.mix_key, keys.data(), size * sizeof(unsigned long long), cudaMemcpyHostToDevice, w->stream));
    CK(cudaMemcpyAsync(d.mix_idx, idx.data(), size * sizeof(uint32_t), cudaMemcpyHostToDevice, w->stream));
    CK(cudaMemcpyAsync(d.mix_mat, mat.data(), (size / 2) * sizeof(float2), cudaMemcpyHostToDevice, w->stream));
    CK(cudaStreamSynchronize(w->stream));
    return B2D_OK;
}
static int mixing_ids_ok(b2d_world *w, uint32_t n, const uint32_t *id0, const uint32_t *id1, const char *fn) {
    if (n && (!id0 || !id1)) { w->error = std::string(fn) + ": NULL id array"; return B2D_ERR_ARGUMENT; }
    for (uint32_t k = 0; k < n; ++k)
        if (id0[k] >= B2D_MATERIAL_UNASSIGNED || id1[k] >= B2D_MATERIAL_UNASSIGNED) {
            w->error = std::string(fn) + ": material ids must be below 0xFFFF"; return B2D_ERR_ARGUMENT;
        }
    return B2D_OK;
}
static uint32_t mixing_key(uint32_t a, uint32_t b) { return a < b ? (a << 16) | b : (b << 16) | a; }     // material_pair_key

int b2d_set_material_mixing(b2d_world *w, uint32_t n, const uint32_t *id0, const uint32_t *id1, const float *friction,
                            const float *restitution) {
    if (!w) return B2D_ERR_ARGUMENT;
    if (int rc = mixing_ids_ok(w, n, id0, id1, "b2d_set_material_mixing")) return rc;
    if (n && (!friction || !restitution)) { w->error = "b2d_set_material_mixing: NULL friction or restitution"; return B2D_ERR_ARGUMENT; }
    if (!n) return B2D_OK;
    cudaSetDevice(w->cfg.device);
    for (uint32_t k = 0; k < n; ++k) w->mixing[mixing_key(id0[k], id1[k])] = make_float2(friction[k], restitution[k]);
    return upload_mixing(w);
}

int b2d_remove_material_mixing(b2d_world *w, uint32_t n, const uint32_t *id0, const uint32_t *id1) {
    if (!w) return B2D_ERR_ARGUMENT;
    if (int rc = mixing_ids_ok(w, n, id0, id1, "b2d_remove_material_mixing")) return rc;
    if (!n) return B2D_OK;
    cudaSetDevice(w->cfg.device);
    size_t erased = 0;
    for (uint32_t k = 0; k < n; ++k) erased += w->mixing.erase(mixing_key(id0[k], id1[k]));
    return erased ? upload_mixing(w) : B2D_OK;
}

// ------------------------------------------------------------------ one step

static int enqueue_broadphase(b2d_world *w) {
    Dev &d = w->d; cudaStream_t s = w->stream;
    if (d.nbodies) {        // first: k_bp_cells also zeroes lmask, which k_bp_separate fills, and newcount
        CK(cudaMemsetAsync(d.cell_box, 0xFF, 6 * sizeof(uint32_t), s));
        LAUNCH(k_bp_cells, d.nbodies, 256, d, d.cellkey, d.cellbody, d.cell_box);
    }
    CK(cudaMemsetAsync(d.mhash_key, 0xFF, (size_t)d.mhash_size * sizeof(unsigned long long), s));
    LAUNCH(k_bp_separate, d.NM, 256, d);
    size_t t = w->cub_tmp_bytes;
    CK(cub::DeviceScan::ExclusiveSum(w->cub_tmp, t, d.free_flag, d.free_rank, (int)d.NM, s)); ++w->launches;
    LAUNCH(k_bp_free_list, d.NM, 256, d);
    if (d.nbodies) {
        LAUNCH(k_bp_cell_mode, d.chash_size, 256, d);            // direct table or cell hash (clears the hash when it is used)
        t = w->cub_tmp_bytes;
        CK(cub::DeviceRadixSort::SortPairs(w->cub_tmp, t, d.cellkey, d.cellkey_s, d.cellbody, d.cellbody_s, (int)d.nbodies, 0, w->cell_key_bits, s)); w->launches += 4;
        LAUNCH(k_bp_cell_starts, d.nbodies, 256, d);
        // a warp per query body while that still fills the machine with few bodies, a thread per body beyond
        const bool bp_warp = d.nbodies <= w->bp_warp_max;
        void (*count_pass)(Dev) = w->bp_half ? k_bp_pairs<false, true> : k_bp_pairs<false, false>;
        if (bp_warp) LAUNCH(k_bp_pairs_warp<false>, (uint64_t)d.nbodies * 32, 256, d); else LAUNCH(count_pass, d.nbodies, 128, d);
        t = w->cub_tmp_bytes;
        CK(cub::DeviceScan::ExclusiveSum(w->cub_tmp, t, d.newcount, d.newoff, (int)d.nbodies, s)); ++w->launches;
        if (bp_warp) LAUNCH(k_bp_pairs_warp<true>, (uint64_t)d.nbodies * 32, 256, d); else LAUNCH(k_bp_pairs<true>, d.nbodies, 128, d);
        LAUNCH(k_bp_append, d.NM, 256, d);
        LAUNCH(k_bp_finish, 1, 32, d);
    }
    return B2D_OK;
}
static int enqueue_narrowphase(b2d_world *w) {
    Dev &d = w->d; cudaStream_t s = w->stream;
    CK(cudaMemsetAsync(d.cnt->npcount, 0, 32 * sizeof(uint32_t), s));        // histogram + cursors
    LAUNCH(k_np_keys, d.NM, 256, d);
    LAUNCH(k_np_scatter, d.NM, 256, d);           // CTAs of exactly 256 threads (window size)
    LAUNCH(k_np_collide_light, d.NM, 128, d);
    LAUNCH(k_np_collide<5>, d.NM, 128, d);
    LAUNCH(k_np_collide<9>, d.NM, 128, d);
    return B2D_OK;
}
// connected components over the current edges (manifolds + joints): island label per body
static int enqueue_cc(b2d_world *w) {
    Dev &d = w->d;
    CK(cudaMemsetAsync(&d.cnt->nislands, 0, sizeof(uint32_t), w->stream));
    LAUNCH(k_cc_init, d.nbodies, 256, d);
    LAUNCH(k_cc_union, (uint64_t)d.NM + d.nhinges, 256, d, 0);
    LAUNCH(k_cc_flatten, d.nbodies, 256, d, 0);
    LAUNCH(k_cc_union, (uint64_t)d.NM + d.nhinges, 256, d, 1);
    LAUNCH(k_cc_flatten, d.nbodies, 256, d, 1);
    w->labels_stale = false;
    return B2D_OK;
}
static int enqueue_islands(b2d_world *w) {
    Dev &d = w->d;
    { int rc = enqueue_cc(w); if (rc) return rc; }
    const uint64_t j = w->updates++;                                 // island_manager::update calls so far
    if (d.sleeping && d.nbodies) {
        // m_last_time inside put_islands_to_sleep is the time of the PREVIOUS update (island_manager.cpp:538, :611-613);
        // update j happens at j * fixed_dt, attach time 0
        const double last_time = j ? double(j - 1) * double(w->cfg.fixed_dt) : 0.0;
        cudaStream_t s = w->stream;
        CK(cudaMemsetAsync(d.size_new, 0, d.nbodies * sizeof(uint32_t), s));
        CK(cudaMemsetAsync(d.isl_flags, 0, d.nbodies * sizeof(uint32_t), s));
        CK(cudaMemsetAsync(d.contributor, 0, d.nbodies * sizeof(unsigned long long), s));
        CK(cudaMemsetAsync(d.heir, 0, d.nbodies * sizeof(unsigned long long), s));
        LAUNCH(k_sleep_gather, d.nbodies, 256, d);
        LAUNCH(k_sleep_heirs, d.nbodies, 256, d);
        LAUNCH(k_sleep_decide, d.nbodies, 256, d, last_time);
        LAUNCH(k_sleep_apply, d.nbodies, 256, d);
        std::swap(d.isl_size, d.size_new);
        std::swap(d.isl_ts, d.ts_new);
    }
    return B2D_OK;
}
// solver.update in three segments so that the velocity solve can be bracketed by timing events between two graphs:
// A gravity .. row preparation, B the velocity iterations, C integration .. refresh.
// solve_restitution, first thing in solver::update (solver.cpp:397): the entity graph as adjacency lists, then one thread per island
static int enqueue_restitution(b2d_world *w) {
    Dev &d = w->d; cudaStream_t s = w->stream;
    if (!d.rest_iters || !d.nbodies) return B2D_OK;
    CK(cudaMemsetAsync(d.rcnt, 0, d.nbodies * sizeof(uint32_t), s));
    CK(cudaMemsetAsync(d.rcur, 0, d.nbodies * sizeof(uint32_t), s));
    CK(cudaMemsetAsync(d.rstamp, 0, d.nbodies * sizeof(uint32_t), s));
    LAUNCH(k_rest_count, (uint64_t)d.NM + d.nhinges, 256, d);
    size_t t = w->cub_tmp_bytes;
    CK(cub::DeviceScan::ExclusiveSum(w->cub_tmp, t, d.rcnt, d.roff, (int)d.nbodies, s)); ++w->launches;
    LAUNCH(k_rest_fill, (uint64_t)d.NM + d.nhinges, 256, d);
    LAUNCH(k_rest_sort, d.nbodies, 128, d);
    LAUNCH(k_rest_solve, d.nbodies, 64, d);
    return B2D_OK;
}
static int enqueue_gravity(b2d_world *w) {
    Dev &d = w->d;
    if (d.nbodies) LAUNCH(k_gravity, d.nbodies, 256, d);
    return B2D_OK;
}
// The island rebuild after the connected components: census, colouring, tile packing, sort keys, sorts and colour
// ranges.  A pure function of the constraint graph (and, on the dataflow path, of the spatial ranks and point counts);
// what it leaves -- parent, btile / bslot, the tile tables, cidx_s / hidx_s, the key arrays and the range counters --
// stays valid for as long as the graph does not change.
static int enqueue_rebuild(b2d_world *w, int recolor) {
    Dev &d = w->d; cudaStream_t s = w->stream;
    CK(cudaMemsetAsync(d.isl_nb, 0, 3 * (size_t)d.NB * sizeof(uint32_t), s));             // island census: bodies, manifolds, joints
    CK(cudaMemsetAsync(d.tile_nb, 0, 5 * (size_t)d.max_tiles * sizeof(uint32_t), s));      // tile body counts and (empty) ranges
    LAUNCH(k_island_census, std::max<uint32_t>(d.nbodies, 1), 256, d);                      // + resets of the colouring / packing accumulators
    LAUNCH(k_color_list, d.NM, 256, d, recolor);
    CK(coop_launch(w, k_color, w->coop_blocks_color, 256, d));
    size_t t;
    if (d.nbodies) {        // island tiles: pack the small islands
        LAUNCH(k_tile_weights, d.nbodies, 256, d);
        t = w->cub_tmp_bytes;
        CK(cub::DeviceScan::ExclusiveSum(w->cub_tmp, t, d.swgt, d.swsum, (int)d.nbodies, s)); ++w->launches;
        LAUNCH(k_tile_assign, d.nbodies, 256, d);
    }
    LAUNCH(k_color_keys, d.NM, 256, d);
    t = w->cub_tmp_bytes;
    CK(cub::DeviceRadixSort::SortPairs(w->cub_tmp, t, d.ckey, d.ckey_s, d.cidx, d.cidx_s, (int)d.NM, 0, COLOR_KEY_BITS, s)); w->launches += 3;
    t = w->cub_tmp_bytes;
    CK(cub::DeviceRadixSort::SortPairs(w->cub_tmp, t, d.hkey, d.hkey_s, d.hidx, d.hidx_s, (int)d.NH, 0, COLOR_KEY_BITS, s)); w->launches += 3;
    LAUNCH(k_color_offsets, d.NM, 256, d);
    LAUNCH(k_color_fixup, 1, 32, d);
    if (d.max_tiles) LAUNCH(k_tile_plan, (uint64_t)d.max_tiles * TILE_CAP, TILE_CAP, d);
    return B2D_OK;
}
static int enqueue_prepare(b2d_world *w) {
    Dev &d = w->d;
    LAUNCH(k_prepare_contacts, d.NM, 256, d);
    if (d.nhinges) LAUNCH(k_prepare_hinges, d.nhinges, 256, d);
    return B2D_OK;
}
static int enqueue_solver_a(b2d_world *w, int recolor) {
    int rc;
    if ((rc = enqueue_restitution(w)) || (rc = enqueue_gravity(w)) || (rc = enqueue_rebuild(w, recolor))) return rc;
    return enqueue_prepare(w);
}
static int enqueue_solver_b(b2d_world *w) {
    Dev &d = w->d;
    const int vi = (int)w->cfg.velocity_iterations;
    // The two schedules work on disjoint islands.  (Forking the tile kernel onto a second stream was measured: no gain --
    // the cooperative launch wants the whole machine and waits for the tiles, or the tiles wait for it.)
    const int pi = (int)w->cfg.position_iterations;
    if (d.max_tiles) {      // the tiled islands' whole solver.update: two-point tiles [0, ntiles2), then the generic ones
        k_island_tiles_2p<<<w->tile_fused_blocks_2p, TILE_CAP, TILE_FUSED_SMEM_2P, w->stream>>>(d, vi, pi); ++w->launches;
        k_island_tiles<<<w->tile_fused_blocks, TILE_CAP, TILE_FUSED_SMEM, w->stream>>>(d, vi, pi); ++w->launches;
    }
    CK(coop_launch(w, k_solve_df, w->coop_blocks_df, B2D_SOLVE_THREADS, d, vi));
    return B2D_OK;
}
static int enqueue_integrate(b2d_world *w) {
    Dev &d = w->d;
    LAUNCH(k_integrate, d.nbodies, 256, d, w->cfg.position_iterations == 0 ? 1 : 0);
    return B2D_OK;
}
static int enqueue_solver_c(b2d_world *w) {
    Dev &d = w->d;
    const int pi = (int)w->cfg.position_iterations;
    LAUNCH(k_store_impulses, d.NM, 256, d);
    if (pi > 0) {
        CK(coop_launch(w, k_position_df, w->coop_blocks_pos_df, B2D_POS_THREADS, d, pi));
        LAUNCH(k_finalize, d.nbodies, 256, d);
    }
    return B2D_OK;
}
static int enqueue_solver(b2d_world *w) {
    const int recolor = ((w->cfg.flags & B2D_FLAG_RECOLOR_EACH_STEP) || w->contacts_dirty) ? 1 : 0;
    w->contacts_dirty = false;
    int rc = enqueue_solver_a(w, recolor); if (rc) return rc;
    ++w->host_rebuilt;
    const int slot = (int)(w->timed_steps % b2d_world::RING);
    if (w->timing) cudaEventRecord(w->ev_solve0[slot], w->stream);
    rc = enqueue_solver_b(w); if (rc) return rc;
    if (w->timing) { cudaEventRecord(w->ev_solve1[slot], w->stream); cudaEventRecord(w->ev_int0[slot], w->stream); }
    rc = enqueue_integrate(w); if (rc) return rc;
    if (w->timing) cudaEventRecord(w->ev_int1[slot], w->stream);
    rc = enqueue_solver_c(w); if (rc) return rc;
    if (w->timing) { ++w->timed_steps; w->timed = true; }
    return B2D_OK;
}

// A hand-over added bodies at the end and / or removed some: the classes of everybody else stand unless the typical
// size moved; departures only ever make the grid pitch an over-estimate.
static int classify_arrivals(b2d_world *w) {
    Dev &d = w->d;
    const float big = w->class_cnt ? float(4.0 * w->class_sum / w->class_cnt) : 1e30f;
    if (std::fabs(big - w->class_big) > 0.1f * w->class_big) return reclassify(w);
    bool grew = false;
    for (uint32_t i = w->class_new_first; i < d.nbodies; ++i) {
        const float dm = w->diam[i];
        if (dm <= 0) continue;
        if (!std::isfinite(dm) || dm > w->class_big) return reclassify(w);
        if (dm > w->max_extent) { w->max_extent = dm; grew = true; }
    }
    if (grew) { d.cell = w->max_extent + 2 * BREAKING_THRESHOLD + 1e-3f; d.inv_cell = 1.0f / d.cell; drop_graphs(w); }
    w->class_new_first = d.nbodies; w->class_removed = false;
    return B2D_OK;
}
// Size the fields of the broadphase cell key to the world as it is now (with room to grow: half the extent again on
// every side, at least 16 cells); runs when the step sequence is (re)captured, i.e. when the population changed.
static int measure_cells(b2d_world *w) {
    Dev &d = w->d;
    if (!d.nbodies) return B2D_OK;
    int *dev6 = (int *)w->stage;
    const int init[6] = {0x7FFFFFFF, 0x7FFFFFFF, 0x7FFFFFFF, -0x7FFFFFFF, -0x7FFFFFFF, -0x7FFFFFFF};
    int ext[6];
    CK(cudaMemcpyAsync(dev6, init, sizeof(init), cudaMemcpyHostToDevice, w->stream));
    LAUNCH(k_cell_extent, d.nbodies, 256, d, dev6);
    CK(cudaMemcpyAsync(ext, dev6, sizeof(ext), cudaMemcpyDeviceToHost, w->stream));
    CK(cudaStreamSynchronize(w->stream));
    int total = 0;
    for (int k = 0; k < 3; ++k) {
        if (ext[k] > ext[3 + k]) { d.cell_org[k] = -(1 << 15); d.cell_bits[k] = 16; total += 16; continue; }
        const long long span = (long long)ext[3 + k] - ext[k] + 1, room = std::max<long long>(16, span / 2);
        int bits = 1;
        while ((1LL << bits) < span + 2 * room + 2 && bits < 16) ++bits;
        d.cell_bits[k] = bits;
        d.cell_org[k] = (int)std::max<long long>(ext[k] - room, -(1LL << 30));
        total += bits;
    }
    w->cell_key_bits = total;
    return B2D_OK;
}
static int prepare_step(b2d_world *w) {
    int rc = B2D_OK;
    if (w->class_dirty) rc = reclassify(w);
    else if (w->class_new_first < w->d.nbodies || w->class_removed) rc = classify_arrivals(w);
    if (rc) return rc;
    if (w->cells_dirty) { rc = measure_cells(w); w->cells_dirty = false; }
    return rc;
}

int b2d_run_phases(b2d_world *w, uint32_t mask) {
    if (!w) return B2D_ERR_ARGUMENT;
    cudaSetDevice(w->cfg.device);
    ++w->state_epoch;
    int rc = prepare_step(w); if (rc) return rc;
    if (mask & B2D_PHASE_BROAD) if ((rc = enqueue_broadphase(w))) return rc;
    if (mask & B2D_PHASE_NARROW) if ((rc = enqueue_narrowphase(w))) return rc;
    if (mask & B2D_PHASE_ISLANDS) if ((rc = enqueue_islands(w))) return rc;
    if (mask & B2D_PHASE_SOLVE) if ((rc = enqueue_solver(w))) return rc;
    CK(cudaGetLastError());
    return B2D_OK;
}

extern "C++" {
#ifndef B2D_EMU
// Capture `body` as the body of a conditional IF node of the graph being captured on w->stream, behind k_rebuild_decide,
// which opens the node iff Counters::graph_changed is set.  The body goes into the node's own graph through a capture on
// w->body_stream (the enqueue_* functions launch on w->stream, which points there meanwhile).
template<typename F>
static int enqueue_if_changed(b2d_world *w, F body) {
    cudaStreamCaptureStatus status; cudaGraph_t g = nullptr; const cudaGraphNode_t *deps = nullptr; size_t ndeps = 0;
    CK(cudaStreamGetCaptureInfo(w->stream, &status, nullptr, &g, &deps, &ndeps));
    cudaGraphConditionalHandle h;
    CK(cudaGraphConditionalHandleCreate(&h, g, 1u, cudaGraphCondAssignDefault));      // rebuild unless told otherwise
    k_rebuild_decide<<<1, 32, 0, w->stream>>>(w->d, h);                                  // control, not counted as a launch
    CK(cudaGetLastError());
    CK(cudaStreamGetCaptureInfo(w->stream, &status, nullptr, &g, &deps, &ndeps));
    cudaGraphNodeParams p = {};
    p.type = cudaGraphNodeTypeConditional;
    p.conditional.handle = h; p.conditional.type = cudaGraphCondTypeIf; p.conditional.size = 1;
    cudaGraphNode_t node;
    CK(cudaGraphAddNode(&node, g, deps, ndeps, &p));
    CK(cudaStreamBeginCaptureToGraph(w->body_stream, p.conditional.phGraph_out[0], nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal));
    cudaStream_t main = w->stream;
    w->stream = w->body_stream;
    const int rc = body();
    w->stream = main;
    cudaGraph_t bg = nullptr;
    const cudaError_t e = cudaStreamEndCapture(w->body_stream, &bg);
    if (rc) return rc;
    CK(e);
    CK(cudaStreamUpdateCaptureDependencies(w->stream, &node, 1, cudaStreamSetCaptureDependencies));
    return B2D_OK;
}
#else
template<typename F>
static int enqueue_if_changed(b2d_world *w, F) { w->error = "conditional graph nodes: not in the CPU emulation"; return B2D_ERR_UNSUPPORTED; }
#endif
// Everything before the velocity solve, as captured.  With `reuse` (only where the step has neither island sleeping nor
// the restitution solver) the connected components and the island rebuild sit under a conditional node that skips them
// while the constraint graph is unchanged; gravity, which neither reads nor writes anything they touch, runs first.
static int enqueue_front(b2d_world *w, bool reuse) {
    int rc;
    if ((rc = enqueue_broadphase(w)) || (rc = enqueue_narrowphase(w))) return rc;
    if (!reuse) { if ((rc = enqueue_islands(w))) return rc; return enqueue_solver_a(w, 0); }
    if ((rc = enqueue_gravity(w))) return rc;
    if ((rc = enqueue_if_changed(w, [&]() { const int r = enqueue_cc(w); return r ? r : enqueue_rebuild(w, 0); }))) return rc;
    return enqueue_prepare(w);
}
// Capture [begin, end) of the step sequence into an executable graph.  Returns false (and leaves the stream usable)
// if the capture is refused; the caller then falls back to plain launches for good.
template<typename F>
static bool capture(b2d_world *w, cudaGraphExec_t &out, bool patchable, F body) {
    const uint64_t launches0 = w->launches, updates0 = w->updates;
    if (cudaStreamBeginCapture(w->stream, cudaStreamCaptureModeThreadLocal) != cudaSuccess) { cudaGetLastError(); return false; }
    const int rc = body();
    cudaGraph_t g = nullptr;
    const cudaError_t e = cudaStreamEndCapture(w->stream, &g);
    w->launches = launches0; w->updates = updates0;                // nothing ran yet
    if (rc != B2D_OK || e != cudaSuccess || !g) { cudaGetLastError(); if (g) cudaGraphDestroy(g); return false; }
    // same kernels in the same order with new arguments / grid sizes (bodies came or went): patch the executable graph in
    // place, which is much cheaper than instantiating a new one.  A graph with a conditional node is instantiated anew:
    // its new handle has to reach both the node and the kernel that sets it.
    if (out && patchable) {
        cudaGraphExecUpdateResultInfo info;
        if (cudaGraphExecUpdate(out, g, &info) == cudaSuccess) { cudaGraphDestroy(g); return true; }
        cudaGetLastError();
    }
    if (out) { cudaGraphExecDestroy(out); out = nullptr; }
    const bool ok = cudaGraphInstantiate(&out, g, 0) == cudaSuccess;
    cudaGraphDestroy(g);
    if (!ok) { cudaGetLastError(); out = nullptr; }
    return ok;
}
static bool build_graphs(b2d_world *w) {
    w->graph_valid = false;
    const bool reuse = w->graph_reuse && w->body_stream && !w->d.sleeping && !w->d.rest_iters;
    uint64_t n_pre = 0, n_solve = 0, n_post = 0;
    auto counted = [&](uint64_t &n, auto fn) { return [&, fn]() { const uint64_t l0 = w->launches; int rc = fn(); n = w->launches - l0; return rc; }; };
    bool ok = capture(w, w->gx_pre, !reuse, counted(n_pre, [&]() { return enqueue_front(w, reuse); }));
    ok = ok && capture(w, w->gx_solve, true, counted(n_solve, [&]() { return enqueue_solver_b(w); }));
    ok = ok && capture(w, w->gx_post, true, counted(n_post, [&]() { return enqueue_solver_c(w); }));
    ok = ok && capture(w, w->gx_all, !reuse, [&]() { int rc; if ((rc = enqueue_front(w, reuse))) return rc;
                                                     if ((rc = enqueue_solver_b(w))) return rc; if ((rc = enqueue_integrate(w))) return rc; return enqueue_solver_c(w); });
    // the driver refused the conditional node: graphs that rebuild the islands every step
    if (!ok && reuse) { destroy_graphs(w); w->graph_reuse = false; return build_graphs(w); }
    if (!ok) { destroy_graphs(w); w->use_graph = false; return false; }
    w->graph_launches = n_pre + n_solve + n_post + 1;
    w->graph_cond = reuse;
    w->graph_valid = true;
    mark_graph_changed(w);          // a new capture starts with a rebuild
    return true;
}
} // extern "C++"

int b2d_step(b2d_world *w, uint32_t num_steps) {
    if (!w) return B2D_ERR_ARGUMENT;
    cudaSetDevice(w->cfg.device);
    ++w->state_epoch;
    int rc = prepare_step(w); if (rc) return rc;
    cudaEventRecord(w->ev_step0, w->stream);
    for (uint32_t i = 0; i < num_steps; ++i) {
        // graphs replay a fixed sequence: island sleeping passes a fresh timestamp every step and a recolouring step
        // runs a different colouring kernel argument, both go the plain way; so does the restitution solver (first version: its
        // per-island thread carries a large local frame, kept out of graph capture)
        const bool plain = !w->use_graph || w->d.sleeping || w->d.rest_iters || w->contacts_dirty || (w->cfg.flags & B2D_FLAG_RECOLOR_EACH_STEP) || w->d.nbodies == 0;
        if (!plain && !w->graph_valid) build_graphs(w);
        if (plain || !w->graph_valid) {
            rc = b2d_run_phases(w, B2D_PHASE_ALL);
            if (rc) return rc;
        } else if (w->timing) {
            const int slot = (int)(w->timed_steps % b2d_world::RING);
            CK(cudaGraphLaunch(w->gx_pre, w->stream));
            cudaEventRecord(w->ev_solve0[slot], w->stream);
            CK(cudaGraphLaunch(w->gx_solve, w->stream));
            cudaEventRecord(w->ev_solve1[slot], w->stream);
            cudaEventRecord(w->ev_int0[slot], w->stream);
            { const uint64_t l0 = w->launches; rc = enqueue_integrate(w); w->launches = l0; if (rc) return rc; }
            cudaEventRecord(w->ev_int1[slot], w->stream);
            CK(cudaGraphLaunch(w->gx_post, w->stream));
            ++w->timed_steps; w->timed = true; ++w->updates;
            w->launches += w->graph_launches;
            if (!w->graph_cond) ++w->host_rebuilt;
        } else {
            CK(cudaGraphLaunch(w->gx_all, w->stream));
            ++w->updates;
            w->launches += w->graph_launches;
            if (!w->graph_cond) ++w->host_rebuilt;
        }
        ++w->steps;
    }
    cudaEventRecord(w->ev_step1, w->stream);
    return B2D_OK;
}

// ------------------------------------------------------------------ state in / out

int b2d_upload_state(b2d_world *w, const float *pos, const float *orn, const float *lv, const float *av) {
    if (!w || !pos || !orn || !lv || !av) return B2D_ERR_ARGUMENT;
    cudaSetDevice(w->cfg.device);
    ++w->state_epoch;
    Dev &d = w->d; const size_t n = d.nbodies; cudaStream_t s = w->stream;
    float *sp = w->stage, *so = sp + 3 * n, *sl = so + 4 * n, *sa = sl + 3 * n;
    CK(cudaMemcpyAsync(sp, pos, 3 * n * sizeof(float), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(so, orn, 4 * n * sizeof(float), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(sl, lv, 3 * n * sizeof(float), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(sa, av, 3 * n * sizeof(float), cudaMemcpyHostToDevice, s));
    LAUNCH(k_unpack_state, n, 256, d, sp, so, sl, sa, (uint32_t)n);
    LAUNCH(k_refresh_bodies, n, 256, d, 0u, (uint32_t)n);
    return B2D_OK;
}

int b2d_download_state(b2d_world *w, float *pos, float *orn, float *lv, float *av, float *bb, float *iw) {
    if (!w) return B2D_ERR_ARGUMENT;
    cudaSetDevice(w->cfg.device);
    Dev &d = w->d; const size_t n = d.nbodies; cudaStream_t s = w->stream;
    float *sp = w->stage, *so = sp + 3 * n, *sl = so + 4 * n, *sa = sl + 3 * n, *sb = sa + 3 * n, *si = sb + 6 * n;
    LAUNCH(k_pack_state, n, 256, d, pos ? sp : nullptr, orn ? so : nullptr, lv ? sl : nullptr, av ? sa : nullptr, bb ? sb : nullptr, iw ? si : nullptr, (uint32_t)n);
    if (pos) CK(cudaMemcpyAsync(pos, sp, 3 * n * sizeof(float), cudaMemcpyDeviceToHost, s));
    if (orn) CK(cudaMemcpyAsync(orn, so, 4 * n * sizeof(float), cudaMemcpyDeviceToHost, s));
    if (lv) CK(cudaMemcpyAsync(lv, sl, 3 * n * sizeof(float), cudaMemcpyDeviceToHost, s));
    if (av) CK(cudaMemcpyAsync(av, sa, 3 * n * sizeof(float), cudaMemcpyDeviceToHost, s));
    if (bb) CK(cudaMemcpyAsync(bb, sb, 6 * n * sizeof(float), cudaMemcpyDeviceToHost, s));
    if (iw) CK(cudaMemcpyAsync(iw, si, 9 * n * sizeof(float), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    return B2D_OK;
}

static int fetch_counters(b2d_world *w, Counters &c) {
    CK(cudaMemcpyAsync(&c, w->d.cnt, sizeof(Counters), cudaMemcpyDeviceToHost, w->stream));
    CK(cudaStreamSynchronize(w->stream));
    return B2D_OK;
}

// Host-side gather of the alive manifolds in slot order (the device arrays have holes).
struct HostManifolds {
    std::vector<uint2> pair; std::vector<uint32_t> state; std::vector<uint32_t> slots;
};
static int fetch_manifolds(b2d_world *w, HostManifolds &hm, uint32_t &hwm) {
    Counters c; int rc = fetch_counters(w, c); if (rc) return rc;
    hwm = c.hwm;
    hm.pair.resize(hwm); hm.state.resize(hwm);
    if (hwm) {
        CK(cudaMemcpyAsync(hm.pair.data(), w->d.mpair, hwm * sizeof(uint2), cudaMemcpyDeviceToHost, w->stream));
        CK(cudaMemcpyAsync(hm.state.data(), w->d.mstate, hwm * sizeof(uint32_t), cudaMemcpyDeviceToHost, w->stream));
        CK(cudaStreamSynchronize(w->stream));
    }
    hm.slots.clear();
    for (uint32_t m = 0; m < hwm; ++m) if (hm.state[m] & MS_ALIVE) hm.slots.push_back(m);
    return B2D_OK;
}

int b2d_num_manifolds(b2d_world *w, uint32_t *n) {
    if (!w || !n) return B2D_ERR_ARGUMENT;
    cudaSetDevice(w->cfg.device);
    HostManifolds hm; uint32_t hwm; int rc = fetch_manifolds(w, hm, hwm); if (rc) return rc;
    *n = (uint32_t)hm.slots.size();
    return B2D_OK;
}

int b2d_download_pairs(b2d_world *w, uint32_t capacity, uint32_t *pairs, uint32_t *n) {
    if (!w || !n) return B2D_ERR_ARGUMENT;
    cudaSetDevice(w->cfg.device);
    HostManifolds hm; uint32_t hwm; int rc = fetch_manifolds(w, hm, hwm); if (rc) return rc;
    *n = (uint32_t)hm.slots.size();
    if (*n > capacity) { w->error = "b2d_download_pairs: capacity too small"; return B2D_ERR_CAPACITY; }
    for (uint32_t k = 0; k < *n; ++k) { pairs[2 * k] = hm.pair[hm.slots[k]].x; pairs[2 * k + 1] = hm.pair[hm.slots[k]].y; }
    return B2D_OK;
}

int b2d_download_contacts(b2d_world *w, uint32_t capacity, uint32_t *pairs, uint32_t *num, float *pt18, uint32_t *ptu2, uint32_t *n) {
    if (!w || !n) return B2D_ERR_ARGUMENT;
    cudaSetDevice(w->cfg.device);
    HostManifolds hm; uint32_t hwm; int rc = fetch_manifolds(w, hm, hwm); if (rc) return rc;
    *n = (uint32_t)hm.slots.size();
    if (*n > capacity) { w->error = "b2d_download_contacts: capacity too small"; return B2D_ERR_CAPACITY; }
    const Dev &d = w->d;
    std::vector<float4> A(4 * (size_t)hwm), B(4 * (size_t)hwm), N(4 * (size_t)hwm), L(4 * (size_t)hwm), I(4 * (size_t)hwm);
    for (int s = 0; s < 4 && hwm; ++s) {
        size_t off = (size_t)s * d.NM, ho = (size_t)s * hwm;
        CK(cudaMemcpyAsync(A.data() + ho, d.pA + off, hwm * sizeof(float4), cudaMemcpyDeviceToHost, w->stream));
        CK(cudaMemcpyAsync(B.data() + ho, d.pB + off, hwm * sizeof(float4), cudaMemcpyDeviceToHost, w->stream));
        CK(cudaMemcpyAsync(N.data() + ho, d.pN + off, hwm * sizeof(float4), cudaMemcpyDeviceToHost, w->stream));
        CK(cudaMemcpyAsync(L.data() + ho, d.pL + off, hwm * sizeof(float4), cudaMemcpyDeviceToHost, w->stream));
        CK(cudaMemcpyAsync(I.data() + ho, d.pI + off, hwm * sizeof(float4), cudaMemcpyDeviceToHost, w->stream));
    }
    CK(cudaStreamSynchronize(w->stream));
    for (uint32_t k = 0; k < *n; ++k) {
        uint32_t m = hm.slots[k];
        pairs[2 * k] = hm.pair[m].x; pairs[2 * k + 1] = hm.pair[m].y;
        uint32_t np = hm.state[m] & MS_NPTS_MASK;
        num[k] = np;
        for (uint32_t s = 0; s < 4; ++s) {
            float *f = pt18 + ((size_t)k * 4 + s) * 18; uint32_t *u = ptu2 + ((size_t)k * 4 + s) * 2;
            if (s >= np) { std::memset(f, 0, 18 * sizeof(float)); u[0] = u[1] = 0; continue; }
            size_t i = (size_t)s * hwm + m;
            f[0] = A[i].x; f[1] = A[i].y; f[2] = A[i].z; f[3] = B[i].x; f[4] = B[i].y; f[5] = B[i].z;
            f[6] = N[i].x; f[7] = N[i].y; f[8] = N[i].z; f[9] = L[i].x; f[10] = L[i].y; f[11] = L[i].z;
            f[12] = A[i].w; f[13] = B[i].w; f[14] = N[i].w; f[15] = I[i].x; f[16] = I[i].y; f[17] = I[i].z;
            uint32_t bits; std::memcpy(&bits, &L[i].w, 4);
            u[0] = bits & 3u; u[1] = bits >> 2;
        }
    }
    return B2D_OK;
}

int b2d_upload_contacts(b2d_world *w, uint32_t n, const uint32_t *pairs, const uint32_t *num, const float *pt18, const uint32_t *ptu2) {
    if (!w) return B2D_ERR_ARGUMENT;
    cudaSetDevice(w->cfg.device);
    ++w->state_epoch;
    Dev &d = w->d;
    if (n > d.NM) { w->error = "b2d_upload_contacts: max_manifolds exceeded"; return B2D_ERR_CAPACITY; }
    std::vector<uint2> pr(n); std::vector<uint32_t> st(n);
    std::vector<float4> A(4 * (size_t)n), B(4 * (size_t)n), N(4 * (size_t)n), L(4 * (size_t)n), I(4 * (size_t)n);
    for (uint32_t k = 0; k < n; ++k) {
        pr[k] = make_uint2(pairs[2 * k], pairs[2 * k + 1]);
        if (num[k] > 4) { w->error = "b2d_upload_contacts: more than 4 points"; return B2D_ERR_ARGUMENT; }
        for (uint32_t s = 0; s < num[k]; ++s) {      // the point layout packs attachment | lifetime << 2 into one word
            const uint32_t *u = ptu2 + ((size_t)k * 4 + s) * 2;
            if (u[0] > 2u) { w->error = "b2d_upload_contacts: normal_attachment > 2"; return B2D_ERR_ARGUMENT; }
            if (u[1] >= (1u << 30)) { w->error = "b2d_upload_contacts: lifetime >= 2^30"; return B2D_ERR_ARGUMENT; }
        }
        st[k] = MS_ALIVE | (COLOR_NONE << MS_COLOR_SHIFT) | num[k];
        for (uint32_t s = 0; s < 4; ++s) {
            const float *f = pt18 + ((size_t)k * 4 + s) * 18; const uint32_t *u = ptu2 + ((size_t)k * 4 + s) * 2;
            size_t i = (size_t)s * n + k;
            uint32_t bits = (u[0] & 3u) | (u[1] << 2); float fb; std::memcpy(&fb, &bits, 4);
            A[i] = make_float4(f[0], f[1], f[2], f[12]); B[i] = make_float4(f[3], f[4], f[5], f[13]);
            N[i] = make_float4(f[6], f[7], f[8], f[14]); L[i] = make_float4(f[9], f[10], f[11], fb);
            I[i] = make_float4(f[15], f[16], f[17], 0);
        }
    }
    cudaStream_t s_ = w->stream;
    CK(cudaMemsetAsync(d.mstate, 0, (size_t)d.NM * sizeof(uint32_t), s_));
    if (n) {
        CK(cudaMemcpyAsync(d.mpair, pr.data(), n * sizeof(uint2), cudaMemcpyHostToDevice, s_));
        CK(cudaMemcpyAsync(d.mstate, st.data(), n * sizeof(uint32_t), cudaMemcpyHostToDevice, s_));
        for (int s = 0; s < 4; ++s) {
            size_t off = (size_t)s * d.NM, ho = (size_t)s * n;
            CK(cudaMemcpyAsync(d.pA + off, A.data() + ho, n * sizeof(float4), cudaMemcpyHostToDevice, s_));
            CK(cudaMemcpyAsync(d.pB + off, B.data() + ho, n * sizeof(float4), cudaMemcpyHostToDevice, s_));
            CK(cudaMemcpyAsync(d.pN + off, N.data() + ho, n * sizeof(float4), cudaMemcpyHostToDevice, s_));
            CK(cudaMemcpyAsync(d.pL + off, L.data() + ho, n * sizeof(float4), cudaMemcpyHostToDevice, s_));
            CK(cudaMemcpyAsync(d.pI + off, I.data() + ho, n * sizeof(float4), cudaMemcpyHostToDevice, s_));
        }
    }
    CK(cudaMemcpyAsync(&d.cnt->hwm, &n, sizeof(uint32_t), cudaMemcpyHostToDevice, s_));
    mark_graph_changed(w);
    CK(cudaStreamSynchronize(s_));
    w->contacts_dirty = true;
    return B2D_OK;
}

int b2d_download_islands(b2d_world *w, uint32_t *label) {
    if (!w || !label) return B2D_ERR_ARGUMENT;
    cudaSetDevice(w->cfg.device);
    CK(cudaMemcpyAsync(label, w->d.parent, w->d.nbodies * sizeof(uint32_t), cudaMemcpyDeviceToHost, w->stream));
    CK(cudaStreamSynchronize(w->stream));
    return B2D_OK;
}

int b2d_download_solver_order(b2d_world *w, uint32_t *hinge_ids, uint32_t *nh, uint32_t *pairs, uint32_t *nm) {
    if (!w || !nh || !nm) return B2D_ERR_ARGUMENT;
    cudaSetDevice(w->cfg.device);
    Counters c; int rc = fetch_counters(w, c); if (rc) return rc;
    const uint32_t na = c.nactive, nhh = c.nhactive;
    if (na > *nm || nhh > *nh) { w->error = "b2d_download_solver_order: capacity too small"; return B2D_ERR_CAPACITY; }
    // the row headers (hdr / hhdr) are not written for tiled constraints: the pairs come from the manifolds themselves
    std::vector<uint2> mp(na ? w->d.NM : 0);
    std::vector<uint32_t> ck(na), hk(nhh), ci(na), hi(nhh);
    if (na) CK(cudaMemcpyAsync(mp.data(), w->d.mpair, w->d.NM * sizeof(uint2), cudaMemcpyDeviceToHost, w->stream));
    if (na) CK(cudaMemcpyAsync(ci.data(), w->d.cidx_s, na * sizeof(uint32_t), cudaMemcpyDeviceToHost, w->stream));
    if (na) CK(cudaMemcpyAsync(ck.data(), w->d.ckey_s, na * sizeof(uint32_t), cudaMemcpyDeviceToHost, w->stream));
    if (nhh) CK(cudaMemcpyAsync(hi.data(), w->d.hidx_s, nhh * sizeof(uint32_t), cudaMemcpyDeviceToHost, w->stream));
    if (nhh) CK(cudaMemcpyAsync(hk.data(), w->d.hkey_s, nhh * sizeof(uint32_t), cudaMemcpyDeviceToHost, w->stream));
    CK(cudaStreamSynchronize(w->stream));
    // The device arrays are tile-major for the tiled islands; the serial sweep that reproduces the per-body order is
    // colour-major (within a colour the constraints touch disjoint dynamic bodies, so their mutual order is immaterial).
    std::vector<uint32_t> oc(na), oh(nhh);
    for (uint32_t i = 0; i < na; ++i) oc[i] = i;
    for (uint32_t i = 0; i < nhh; ++i) oh[i] = i;
    auto colour = [](uint32_t key) { return (key & KEY_DF) ? (key >> KEY_DF_COLOR_SHIFT) & 63u : key & 63u; };
    std::stable_sort(oc.begin(), oc.end(), [&](uint32_t x, uint32_t y) { return colour(ck[x]) < colour(ck[y]); });
    std::stable_sort(oh.begin(), oh.end(), [&](uint32_t x, uint32_t y) { return colour(hk[x]) < colour(hk[y]); });
    for (uint32_t i = 0; i < na; ++i) { const uint2 p = mp[ci[oc[i]]]; pairs[2 * i] = p.x; pairs[2 * i + 1] = p.y; }
    for (uint32_t i = 0; i < nhh; ++i) hinge_ids[i] = hi[oh[i]];
    *nm = na; *nh = nhh;
    return B2D_OK;
}

int b2d_download_hinge_impulses(b2d_world *w, float *imp5) {
    if (!w || !imp5) return B2D_ERR_ARGUMENT;
    cudaSetDevice(w->cfg.device);
    CK(cudaMemcpyAsync(imp5, w->d.himp, 5 * (size_t)w->d.nhinges * sizeof(float), cudaMemcpyDeviceToHost, w->stream));
    CK(cudaStreamSynchronize(w->stream));
    return B2D_OK;
}

int b2d_get_stats(b2d_world *w, b2d_stats *out) {
    if (!w || !out) return B2D_ERR_ARGUMENT;
    cudaSetDevice(w->cfg.device);
    Dev &d = w->d;
    CK(cudaMemsetAsync(&d.cnt->npoints, 0, sizeof(uint32_t), w->stream));
    LAUNCH(k_count_points, d.NM, 256, d); --w->launches;
    Counters c; int rc = fetch_counters(w, c); if (rc) return rc;
    HostManifolds hm; uint32_t hwm; rc = fetch_manifolds(w, hm, hwm); if (rc) return rc;
    std::memset(out, 0, sizeof(*out));
    out->bodies = d.nbodies; out->manifolds = (uint32_t)hm.slots.size(); out->contact_points = c.npoints; out->hinges = d.nhinges;
    out->contact_colors = c.ncolors_all; out->hinge_colors = c.nhcolors_all; out->islands = c.nislands; out->manifold_high_water = c.hwm;
    out->kernel_launches = w->launches; out->steps = w->steps; out->error_flags = c.err;
    out->steps_rebuilt = w->host_rebuilt + c.steps_rebuilt; out->steps_reused = c.steps_reused;
    if (w->timed && w->timed_steps) {
        // average over the steps since b2d_reset_timers (at most the ring size)
        const uint64_t cnt = std::min<uint64_t>(w->timed_steps, b2d_world::RING);
        double ss = 0, si = 0;
        for (uint64_t k = 0; k < cnt; ++k) {
            int slot = (int)((w->timed_steps - 1 - k) % b2d_world::RING);
            float a = 0, b = 0;
            cudaEventElapsedTime(&a, w->ev_solve0[slot], w->ev_solve1[slot]);
            cudaEventElapsedTime(&b, w->ev_int0[slot], w->ev_int1[slot]);
            ss += a; si += b;
        }
        out->solve_ms = (float)(ss / cnt); out->integrate_ms = (float)(si / cnt);
        if (cudaEventQuery(w->ev_step1) == cudaSuccess) cudaEventElapsedTime(&out->last_step_ms, w->ev_step0, w->ev_step1);
        cudaGetLastError();
    }
    return B2D_OK;
}

// development aid: raw copy of the device counters block
int b2d_debug_counters(b2d_world *w, void *out, uint32_t bytes) {
    if (!w) return B2D_ERR_ARGUMENT;
    cudaSetDevice(w->cfg.device);
    CK(cudaStreamSynchronize(w->stream));
    CK(cudaMemcpy(out, w->d.cnt, std::min<size_t>(bytes, sizeof(Counters)), cudaMemcpyDeviceToHost));
    return B2D_OK;
}
// development aid: the last broadphase's newcount
int b2d_debug_newcount(b2d_world *w, uint32_t *counts) {
    if (!w || !counts) return B2D_ERR_ARGUMENT;
    cudaSetDevice(w->cfg.device);
    CK(cudaStreamSynchronize(w->stream));
    if (w->d.nbodies) CK(cudaMemcpy(counts, w->d.newcount, w->d.nbodies * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    return B2D_OK;
}
// development aid: island tiles of the last step: out = {tiles, tiled manifolds, tiled hinges, manifolds with rows, hinges with rows, max bodies per tile}
int b2d_debug_tiles(b2d_world *w, uint32_t *out6) {
    if (!w || !out6) return B2D_ERR_ARGUMENT;
    cudaSetDevice(w->cfg.device);
    Counters c; int rc = fetch_counters(w, c); if (rc) return rc;
    std::vector<uint32_t> nb(std::min(c.ntiles, w->d.max_tiles));
    if (!nb.empty()) CK(cudaMemcpy(nb.data(), w->d.tile_nb, nb.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    out6[0] = c.ntiles; out6[1] = c.ntiled; out6[2] = c.nhtiled; out6[3] = c.nactive; out6[4] = c.nhactive;
    out6[5] = nb.empty() ? 0u : *std::max_element(nb.begin(), nb.end());
    return B2D_OK;
}
// development aid: the island-tile packing of the last rebuild, as the solve reads it (include/b2d.h)
int b2d_debug_tile_map(b2d_world *w, uint32_t *counts5, uint32_t *btile, uint32_t *bslot, uint32_t *tiles5,
                       uint32_t *tiled_pairs, uint32_t *tiled_hinges) {
    if (!w || !counts5) return B2D_ERR_ARGUMENT;
    cudaSetDevice(w->cfg.device);
    const Dev &d = w->d;
    Counters c; int rc = fetch_counters(w, c); if (rc) return rc;
    const uint32_t nt = std::min(c.ntiles, d.max_tiles), ntc = std::min(c.ntiled, d.NM), nth = std::min(c.nhtiled, d.NH);
    counts5[0] = nt; counts5[1] = std::min(c.ntiles2, nt); counts5[2] = ntc; counts5[3] = nth; counts5[4] = d.max_tiles;
    if (btile && d.nbodies) CK(cudaMemcpy(btile, d.btile, d.nbodies * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    if (bslot && d.nbodies) CK(cudaMemcpy(bslot, d.bslot, d.nbodies * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    if (tiles5 && nt) {
        const uint32_t *src[5] = {d.tile_nb, d.tile_c0, d.tile_c1, d.tile_h0, d.tile_h1};
        for (int k = 0; k < 5; ++k) CK(cudaMemcpy(tiles5 + (size_t)k * nt, src[k], nt * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    }
    if (tiled_pairs && ntc) {
        std::vector<uint32_t> ci(ntc);
        std::vector<uint2> mp(d.NM);
        CK(cudaMemcpy(ci.data(), d.cidx_s, ntc * sizeof(uint32_t), cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(mp.data(), d.mpair, d.NM * sizeof(uint2), cudaMemcpyDeviceToHost));
        for (uint32_t i = 0; i < ntc; ++i) { tiled_pairs[2 * i] = mp[ci[i]].x; tiled_pairs[2 * i + 1] = mp[ci[i]].y; }
    }
    if (tiled_hinges && nth) CK(cudaMemcpy(tiled_hinges, d.hidx_s, nth * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    return B2D_OK;
}
int b2d_reset_timers(b2d_world *w) { if (!w) return B2D_ERR_ARGUMENT; w->timed_steps = 0; return B2D_OK; }

int b2d_set_halo_margin(b2d_world *w, float margin) {
    if (!w || !(margin >= 0.0f)) return B2D_ERR_ARGUMENT;
    w->d.halo_margin = std::max(margin, HALO_MARGIN);
    return B2D_OK;
}
int b2d_device_bounds(b2d_world *w, float *device_out8) {
    if (!w || !device_out8) return B2D_ERR_ARGUMENT;
    cudaSetDevice(w->cfg.device);
    Dev &d = w->d;
    LAUNCH(k_bounds_init, 1, 32, d);
    LAUNCH(k_bounds_reduce, d.nbodies, 256, d);
    LAUNCH(k_bounds_final, 1, 32, d, device_out8);
    CK(cudaGetLastError());
    return B2D_OK;
}

// ------------------------------------------------------------------ raycast

// Enqueue the rebuild of the raycast index if the state changed since the last one; the buffers are allocated by the
// first raycast, so worlds that never query pay nothing.  No host synchronisation (after the first allocation).
static int ray_index(b2d_world *w) {
    Dev &d = w->d; RayIndex &x = w->rx; cudaStream_t s = w->stream;
    if (!w->ray_alloc) {
        const uint32_t NB = d.NB;
        x.hsize = pow2_at_least(2ull * NB);
        const bool ok = dalloc(w, x.key, NB) && dalloc(w, x.key_s, NB) && dalloc(w, x.body, NB) && dalloc(w, x.body_s, NB) &&
                        dalloc(w, x.hkey, x.hsize, 0xFF) && dalloc(w, x.hval, x.hsize) && dalloc(w, x.extra, (size_t)NB + 1) &&
                        dalloc(w, x.bounds, 6);
        if (!ok) return B2D_ERR_CUDA;
        w->ray_alloc = true;
    }
    if (w->ray_epoch == w->state_epoch) return B2D_OK;
    LAUNCH(k_ray_reset, 1, 32, x);
    if (d.nbodies) {
        LAUNCH(k_bp_cells, d.nbodies, 256, d, x.key, x.body, (uint32_t *)nullptr);
        LAUNCH(k_ray_classify, d.nbodies, 256, d, x);
        size_t t = w->cub_tmp_bytes;
        CK(cub::DeviceRadixSort::SortPairs(w->cub_tmp, t, x.key, x.key_s, x.body, x.body_s, (int)d.nbodies, 0, w->cell_key_bits, s)); w->launches += 4;
        CK(cudaMemsetAsync(x.hkey, 0xFF, (size_t)x.hsize * sizeof(unsigned long long), s));
        LAUNCH(k_ray_cell_starts, d.nbodies, 256, d, x);
    }
    CK(cudaGetLastError());
    w->ray_epoch = w->state_epoch;
    return B2D_OK;
}
// Device scratch of at least `bytes` for the rays of the host-array path and the shared ignore list.
static void *ray_scratch(b2d_world *w, size_t bytes) {
    if (bytes <= w->ray_buf_bytes) return w->ray_buf;
    if (w->ray_buf) { cudaStreamSynchronize(w->stream); cudaFree(w->ray_buf); w->ray_buf = nullptr; w->ray_buf_bytes = 0; }
    const size_t want = std::max<size_t>(bytes, 1 << 16);
    if (cudaMalloc(&w->ray_buf, want) != cudaSuccess) { cudaGetLastError(); w->ray_buf = nullptr; w->error = "raycast: cudaMalloc failed"; return nullptr; }
    w->ray_buf_bytes = want;
    return w->ray_buf;
}
static bool ray_args(b2d_world *w, uint32_t n, const float *p0, const float *p1, const uint32_t *ignore_list, uint32_t nignore) {
    if (!w) return false;
    if ((n && (!p0 || !p1)) || (nignore && !ignore_list)) { w->error = "b2d_raycast: missing segment or ignore array"; return false; }
    return true;
}
static std::vector<uint32_t> ray_ignore(const uint32_t *list, uint32_t n) {     // sorted for the kernel's binary search
    std::vector<uint32_t> v(list, list + n);
    std::sort(v.begin(), v.end());
    v.erase(std::unique(v.begin(), v.end()), v.end());
    return v;
}

int b2d_raycast(b2d_world *w, uint32_t n, const float *p0, const float *p1, const uint32_t *ignore_body,
                const uint32_t *ignore_list, uint32_t nignore, uint32_t *body, float *fraction, float *normal, uint32_t *feature) {
    if (!ray_args(w, n, p0, p1, ignore_list, nignore)) return B2D_ERR_ARGUMENT;
    cudaSetDevice(w->cfg.device);
    int rc = ray_index(w); if (rc) return rc;
    if (!n) return B2D_OK;
    const std::vector<uint32_t> ign = ray_ignore(ignore_list, nignore);
    const size_t m = ign.size();
    uint32_t *buf = (uint32_t *)ray_scratch(w, (13 * (size_t)n + m) * sizeof(uint32_t));
    if (!buf) return B2D_ERR_CUDA;
    float *dp0 = (float *)buf, *dp1 = dp0 + 3 * (size_t)n;
    uint32_t *dib = (uint32_t *)(dp1 + 3 * (size_t)n), *dil = dib + n, *dbody = dil + m;
    float *dfr = (float *)(dbody + n), *dnrm = dfr + n;
    uint32_t *dfeat = (uint32_t *)(dnrm + 3 * (size_t)n);
    cudaStream_t s = w->stream;
    CK(cudaMemcpyAsync(dp0, p0, 3 * (size_t)n * sizeof(float), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(dp1, p1, 3 * (size_t)n * sizeof(float), cudaMemcpyHostToDevice, s));
    if (ignore_body) CK(cudaMemcpyAsync(dib, ignore_body, (size_t)n * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
    if (m) CK(cudaMemcpyAsync(dil, ign.data(), m * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
    LAUNCH(k_ray_cast, n, 128, w->d, w->rx, n, dp0, dp1, ignore_body ? dib : nullptr, m ? dil : nullptr, (uint32_t)m, dbody, dfr, dnrm, dfeat);
    CK(cudaGetLastError());
    if (body) CK(cudaMemcpyAsync(body, dbody, (size_t)n * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    if (fraction) CK(cudaMemcpyAsync(fraction, dfr, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, s));
    if (normal) CK(cudaMemcpyAsync(normal, dnrm, 3 * (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, s));
    if (feature) CK(cudaMemcpyAsync(feature, dfeat, (size_t)n * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    return B2D_OK;
}

int b2d_raycast_device(b2d_world *w, uint32_t n, const float *p0, const float *p1, const uint32_t *ignore_body,
                       const uint32_t *ignore_list, uint32_t nignore, uint32_t *body, float *fraction, float *normal, uint32_t *feature) {
    if (!ray_args(w, n, p0, p1, ignore_list, nignore)) return B2D_ERR_ARGUMENT;
    cudaSetDevice(w->cfg.device);
    int rc = ray_index(w); if (rc) return rc;
    if (!n) return B2D_OK;
    const std::vector<uint32_t> ign = ray_ignore(ignore_list, nignore);
    uint32_t *dil = nullptr;
    if (!ign.empty()) {
        dil = (uint32_t *)ray_scratch(w, ign.size() * sizeof(uint32_t));
        if (!dil) return B2D_ERR_CUDA;
        CK(cudaMemcpyAsync(dil, ign.data(), ign.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, w->stream));
    }
    LAUNCH(k_ray_cast, n, 128, w->d, w->rx, n, p0, p1, ignore_body, dil, (uint32_t)ign.size(), body, fraction, normal, feature);
    CK(cudaGetLastError());
    return B2D_OK;
}


// ------------------------------------------------------------------ presentation (k_presentation)

static int enqueue_presentation(b2d_world *w, int mode, float dt, float *out_pos, float *out_orn) {
    cudaSetDevice(w->cfg.device);
    Dev &d = w->d;
    if (d.nbodies) LAUNCH(k_presentation, d.nbodies, 256, d, mode, dt, out_pos, out_orn, d.nbodies);
    CK(cudaGetLastError());
    return B2D_OK;
}
int b2d_update_presentation(b2d_world *w, float interpolation_dt) {
    if (!w) return B2D_ERR_ARGUMENT;
    return enqueue_presentation(w, PRESENT_UPDATE, interpolation_dt, nullptr, nullptr);
}
int b2d_snap_presentation(b2d_world *w) {
    if (!w) return B2D_ERR_ARGUMENT;
    return enqueue_presentation(w, PRESENT_SNAP, 0.0f, nullptr, nullptr);
}
int b2d_download_presentation(b2d_world *w, float *pos, float *orn) {
    if (!w || (!pos && !orn)) return B2D_ERR_ARGUMENT;
    const size_t n = w->d.nbodies;
    float *sp = w->stage, *so = sp + 3 * n;
    if (int rc = enqueue_presentation(w, PRESENT_READ, 0.0f, pos ? sp : nullptr, orn ? so : nullptr)) return rc;
    cudaStream_t s = w->stream;
    if (pos && n) CK(cudaMemcpyAsync(pos, sp, 3 * n * sizeof(float), cudaMemcpyDeviceToHost, s));
    if (orn && n) CK(cudaMemcpyAsync(orn, so, 4 * n * sizeof(float), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    return B2D_OK;
}
int b2d_download_presentation_device(b2d_world *w, float *device_pos, float *device_orn) {
    if (!w || (!device_pos && !device_orn)) return B2D_ERR_ARGUMENT;
    return enqueue_presentation(w, PRESENT_READ, 0.0f, device_pos, device_orn);
}

int b2d_set_timing(b2d_world *w, int enabled) { if (!w) return B2D_ERR_ARGUMENT; w->timing = enabled != 0; return B2D_OK; }

// ------------------------------------------------------------------ dirty-subset staging

int b2d_upload_bodies(b2d_world *w, uint32_t n, const uint32_t *ids, const b2d_body_patch *p) {
    if (!w || !p || (n && !ids)) return B2D_ERR_ARGUMENT;
    cudaSetDevice(w->cfg.device);
    ++w->state_epoch;
    Dev &d = w->d;
    if (!n) return B2D_OK;
    for (uint32_t k = 0; k < n; ++k) {
        if (ids[k] >= d.nbodies) { w->error = "b2d_upload_bodies: body id out of range"; return B2D_ERR_ARGUMENT; }
        if (p->kind && p->kind[k] > B2D_STATIC) { w->error = "b2d_upload_bodies: bad body kind"; return B2D_ERR_ARGUMENT; }
        if (p->material && p->material[k] > B2D_MATERIAL_UNASSIGNED && p->material[k] != B2D_MATERIAL_NONE) {
            w->error = "b2d_upload_bodies: material must be an id up to 0xFFFF or B2D_MATERIAL_NONE"; return B2D_ERR_ARGUMENT;
        }
    }
    if (p->material) {          // a body's points keep the constraint type they were created with: no sensor toggling
        std::vector<uint32_t> flags(d.nbodies);
        CK(cudaMemcpyAsync(flags.data(), d.flags, d.nbodies * sizeof(uint32_t), cudaMemcpyDeviceToHost, w->stream));
        CK(cudaStreamSynchronize(w->stream));
        for (uint32_t k = 0; k < n; ++k)
            if (((flags[ids[k]] & F_SENSOR) != 0) != (p->material[k] == B2D_MATERIAL_NONE)) {
                w->error = "b2d_upload_bodies: a body cannot change between sensor (B2D_MATERIAL_NONE) and material"; return B2D_ERR_UNSUPPORTED;
            }
    }
    if ((size_t)n * 31 > w->stage_floats) { w->error = "b2d_upload_bodies: patch larger than the staging buffer"; return B2D_ERR_CAPACITY; }
    cudaStream_t s = w->stream;
    float *cur = w->stage;
    auto put = [&](const void *host, size_t words) -> const float * {
        if (!host) return nullptr;
        float *dst = cur; cur += words;
        cudaMemcpyAsync(dst, host, words * sizeof(float), cudaMemcpyHostToDevice, s);
        return dst;
    };
    const uint32_t *dev_ids = (const uint32_t *)put(ids, n);
    Patch q;
    q.pos = put(p->pos, 3 * (size_t)n); q.orn = put(p->orn, 4 * (size_t)n); q.linvel = put(p->linvel, 3 * (size_t)n); q.angvel = put(p->angvel, 3 * (size_t)n);
    q.inv_mass = put(p->inv_mass, n); q.inv_inertia = put(p->inv_inertia, 9 * (size_t)n); q.gravity = put(p->gravity, 3 * (size_t)n);
    q.friction = put(p->friction, n); q.restitution = put(p->restitution, n); q.kind = (const uint32_t *)put(p->kind, n);
    q.material = (const uint32_t *)put(p->material, n);
    LAUNCH(k_patch_bodies, n, 256, d, dev_ids, n, q);
    if (p->kind) mark_graph_changed(w);              // body kinds decide the islands and which constraints have rows
    CK(cudaStreamSynchronize(s));                    // the host arrays may be reused by the caller
    if (p->kind) {
        for (uint32_t k = 0; k < n; ++k) w->isdyn[ids[k]] = p->kind[k] == B2D_DYNAMIC ? 1 : 0;
        w->class_dirty = true;
        // a constraint coloured while one of its bodies was not dynamic only avoided the other body's colours: a body
        // that becomes dynamic would bring clashing colours along, so the next step colours everything afresh
        w->contacts_dirty = true;
    }
    return B2D_OK;
}

// ------------------------------------------------------------------ multi-GPU: names, halo, plan, hand-over

int b2d_set_entities(b2d_world *w, uint32_t first, uint32_t n, const uint32_t *entity) {
    if (!w || (n && !entity)) return B2D_ERR_ARGUMENT;
    cudaSetDevice(w->cfg.device);
    Dev &d = w->d;
    if ((uint64_t)first + n > d.nbodies) { w->error = "b2d_set_entities: body id out of range"; return B2D_ERR_ARGUMENT; }
    if (!n) return B2D_OK;
    uint32_t *tmp = (uint32_t *)w->stage;
    CK(cudaMemcpyAsync(tmp, entity, n * sizeof(uint32_t), cudaMemcpyHostToDevice, w->stream));
    LAUNCH(k_entities_set, n, 256, d, first, n, (const uint32_t *)tmp);
    CK(cudaStreamSynchronize(w->stream));
    w->ehash_dirty = true;
    return B2D_OK;
}
int b2d_download_entities(b2d_world *w, uint32_t *entity) {
    if (!w || !entity) return B2D_ERR_ARGUMENT;
    cudaSetDevice(w->cfg.device);
    CK(cudaMemcpyAsync(entity, w->d.entity, w->d.nbodies * sizeof(uint32_t), cudaMemcpyDeviceToHost, w->stream));
    CK(cudaStreamSynchronize(w->stream));
    return B2D_OK;
}

int b2d_island_halo(b2d_world *w, const float *device_boxes, uint32_t nboxes, uint32_t self, uint64_t peer_mask,
                    void *device_records, uint32_t capacity, uint32_t *device_count) {
    if (!w || !device_boxes || !device_records || !device_count || nboxes > 64 || self >= nboxes) return B2D_ERR_ARGUMENT;
    cudaSetDevice(w->cfg.device);
    Dev &d = w->d;
    if (w->labels_stale) { int rc = enqueue_cc(w); if (rc) return rc; }
    CK(cudaMemsetAsync(device_count, 0, sizeof(uint32_t), w->stream));
    if (d.nbodies) {
        LAUNCH(k_ibox_init, d.nbodies, 256, d);
        LAUNCH(k_ibox_reduce, d.nbodies, 256, d);
        LAUNCH(k_halo_collect, d.nbodies, 256, d, device_boxes, nboxes, self, (unsigned long long)peer_mask, (HaloRec *)device_records, capacity, device_count);
    }
    CK(cudaGetLastError());
    return B2D_OK;
}

int b2d_handover_plan(b2d_world *w, const void *device_records, uint32_t my_begin, uint32_t my_end, uint32_t nranks, uint32_t *counts) {
    if (!w || !counts || nranks == 0 || nranks > 64 || my_end < my_begin || (my_end > my_begin && !device_records)) return B2D_ERR_ARGUMENT;
    cudaSetDevice(w->cfg.device);
    Dev &d = w->d; cudaStream_t s = w->stream;
    Trace tr("plan");
    CK(cudaMemsetAsync(w->dev_counts, 0, 4 * 64 * sizeof(uint32_t), s));
    if (my_end > my_begin && my_begin > 0)
        LAUNCH(k_plan_islands, (uint64_t)(my_end - my_begin) * my_begin, 256, d, (const HaloRec *)device_records, my_begin, my_end);
    if (d.nbodies) {
        LAUNCH(k_plan_bodies, d.nbodies, 256, d, w->dev_counts);
        LAUNCH(k_plan_constraints, (uint64_t)d.NM + d.nhinges, 256, d, w->dev_counts);
    }
    w->plan_counts.assign(4 * (size_t)nranks, 0);
    w->host_bdst.resize(d.nbodies);
    CK(cudaMemcpyAsync(w->plan_counts.data(), w->dev_counts, 4 * nranks * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    if (d.nbodies) CK(cudaMemcpyAsync(w->host_bdst.data(), d.bdst, d.nbodies * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    // collision_exclusion between two movers travels with them
    for (uint64_t k : w->exclusions) {
        const uint32_t a = (uint32_t)(k >> 32), b = (uint32_t)k;
        if (a < d.nbodies && b < d.nbodies && w->host_bdst[a] != NO_RANK && w->host_bdst[a] == w->host_bdst[b] && w->host_bdst[a] < nranks) ++w->plan_counts[4 * w->host_bdst[a] + 3];
    }
    w->plan_ranks = nranks;
    tr.mark("done");
    std::memcpy(counts, w->plan_counts.data(), 4 * nranks * sizeof(uint32_t));
    return B2D_OK;
}

uint64_t b2d_handover_bytes(const uint32_t *c) {
    if (!c) return 0;
    uint64_t b = sizeof(BlobHeader) + 16ull * (BLOB_BODY_F4 * (uint64_t)c[0] + BLOB_MANIFOLD_F4 * (uint64_t)c[1] + BLOB_HINGE_F4 * (uint64_t)c[2]) + 8ull * c[3];
    return (b + 15) & ~15ull;
}

int b2d_handover_pack(b2d_world *w, uint32_t dst, void *device_blob, uint64_t capacity) {
    if (!w || !device_blob || dst >= w->plan_ranks) return B2D_ERR_ARGUMENT;
    cudaSetDevice(w->cfg.device);
    ++w->state_epoch;
    Dev &d = w->d; cudaStream_t s = w->stream;
    const uint32_t *c = &w->plan_counts[4 * dst];
    Trace tr("pack");
    if (capacity < b2d_handover_bytes(c)) { w->error = "b2d_handover_pack: blob too small"; return B2D_ERR_CAPACITY; }
    std::vector<uint32_t> ids; ids.reserve(c[0]);
    for (uint32_t i = 0; i < d.nbodies; ++i) if (w->host_bdst[i] == dst) ids.push_back(i);
    // exclusions among the movers travel with them; the local entries stay behind as garbage (ids are never reused) and
    // are dropped from the host list in one sweep
    std::vector<uint2> ex;
    if (c[3]) {
        size_t keep = 0;
        for (uint64_t k : w->exclusions) {
            const uint32_t a = (uint32_t)(k >> 32), b = (uint32_t)k;
            if (a < d.nbodies && b < d.nbodies && w->host_bdst[a] == dst && w->host_bdst[b] == dst) ex.push_back(make_uint2(a, b)); else w->exclusions[keep++] = k;
        }
        w->exclusions.resize(keep);
    }
    if (ids.size() != c[0] || ex.size() != c[3]) { w->error = "b2d_handover_pack: plan is stale"; return B2D_ERR_ARGUMENT; }
    char *blob = (char *)device_blob;
    BlobHeader *hdr = (BlobHeader *)blob;
    float4 *ob = (float4 *)(blob + sizeof(BlobHeader)), *om = ob + (size_t)BLOB_BODY_F4 * c[0], *oh = om + (size_t)BLOB_MANIFOLD_F4 * c[1];
    uint2 *ox = (uint2 *)(oh + (size_t)BLOB_HINGE_F4 * c[2]);
    k_pack_header<<<1, 32, 0, s>>>(hdr, c[0], c[1], c[2], c[3]); ++w->launches;
    if ((size_t)c[0] + 2 * (size_t)c[3] + 4 > w->stage_floats) { w->error = "b2d_handover_pack: plan larger than the staging buffer"; return B2D_ERR_CAPACITY; }
    uint32_t *dev_ids = (uint32_t *)w->stage; uint2 *dev_ex = (uint2 *)(w->stage + ((c[0] + 1u) & ~1u));      // scratch inside the staging buffer
    if (c[0]) {
        CK(cudaMemcpyAsync(dev_ids, ids.data(), c[0] * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
        LAUNCH(k_pack_bodies, c[0], 256, d, (const uint32_t *)dev_ids, c[0], ob);
    }
    size_t t;
    if (c[1]) {
        LAUNCH(k_pack_flag_manifolds, d.NM, 256, d, dst);
        t = w->cub_tmp_bytes;
        CK(cub::DeviceScan::ExclusiveSum(w->cub_tmp, t, d.free_flag, d.free_rank, (int)d.NM, s)); ++w->launches;
        LAUNCH(k_pack_manifolds, d.NM, 256, d, om);
    }
    if (c[2]) {
        LAUNCH(k_pack_flag_hinges, d.NH, 256, d, dst);
        t = w->cub_tmp_bytes;
        CK(cub::DeviceScan::ExclusiveSum(w->cub_tmp, t, d.hidx, d.hidx_s, (int)d.NH, s)); ++w->launches;
        LAUNCH(k_pack_hinges, d.nhinges, 256, d, oh);
    }
    if (c[3]) {
        CK(cudaMemcpyAsync(dev_ex, ex.data(), c[3] * sizeof(uint2), cudaMemcpyHostToDevice, s));
        LAUNCH(k_pack_exclusions, c[3], 256, d, (const uint2 *)dev_ex, c[3], ox);
    }
    // registry.destroy of the local copies: the bodies turn into removed slots, their manifolds and joints die with them
    if (c[0]) {
        LAUNCH(k_remove_bodies, c[0], 256, d, (const uint32_t *)dev_ids, c[0]);
        if (d.nhinges) LAUNCH(k_remove_hinges, d.nhinges, 256, d);
    }
    tr.mark("enqueued");
    CK(cudaStreamSynchronize(s));
    tr.mark("synced");
    for (uint32_t i : ids) { class_forget(w, i); w->host_bdst[i] = NO_RANK; }
    w->class_removed = true; w->ehash_dirty = true; w->labels_stale = true;
    drop_graphs(w);
    return B2D_OK;
}

int b2d_handover_unpack(b2d_world *w, const void *device_blob, uint64_t bytes, uint32_t *counts_out) {
    if (!w || !device_blob || bytes < sizeof(BlobHeader)) return B2D_ERR_ARGUMENT;
    cudaSetDevice(w->cfg.device);
    ++w->state_epoch;
    Dev &d = w->d; cudaStream_t s = w->stream;
    BlobHeader h;
    Trace tr("unpack");
    CK(cudaMemcpyAsync(&h, device_blob, sizeof(h), cudaMemcpyDeviceToHost, s));
    Counters cn; { int rc = fetch_counters(w, cn); if (rc) return rc; }
    tr.mark("blob header on the host (the receive has landed)");
    if (h.magic != BLOB_MAGIC) { w->error = "b2d_handover_unpack: not a hand-over blob"; return B2D_ERR_ARGUMENT; }
    const uint32_t c[4] = {h.nb, h.nm, h.nh, h.nx};
    if (bytes < b2d_handover_bytes(c)) { w->error = "b2d_handover_unpack: blob truncated"; return B2D_ERR_ARGUMENT; }
    if ((uint64_t)d.nbodies + h.nb > d.NB) { w->error = "b2d_handover_unpack: max_bodies exceeded"; return B2D_ERR_CAPACITY; }
    if ((uint64_t)cn.hwm + h.nm > d.NM) { w->error = "b2d_handover_unpack: max_manifolds exceeded"; return B2D_ERR_CAPACITY; }
    if ((uint64_t)d.nhinges + h.nh > w->cfg.max_hinges) { w->error = "b2d_handover_unpack: max_hinges exceeded"; return B2D_ERR_CAPACITY; }
    const char *blob = (const char *)device_blob;
    const float4 *ib = (const float4 *)(blob + sizeof(BlobHeader)), *im = ib + (size_t)BLOB_BODY_F4 * h.nb, *ih = im + (size_t)BLOB_MANIFOLD_F4 * h.nm;
    const uint2 *ix = (const uint2 *)(ih + (size_t)BLOB_HINGE_F4 * h.nh);
    const uint32_t first = d.nbodies;
    d.nbodies = first + h.nb;                       // the entity table below must see the newcomers' slots as live
    if (w->ehash_dirty) {
        CK(cudaMemsetAsync(d.ehash, 0xFF, (size_t)d.ehash_size * sizeof(unsigned long long), s));
        if (first) { Dev old = d; old.nbodies = first; LAUNCH(k_ehash_build, first, 256, old); }
        w->ehash_dirty = false;
    }
    if (h.nb) {
        LAUNCH(k_unpack_bodies, h.nb, 256, d, first, h.nb, ib);
        LAUNCH(k_refresh_bodies, h.nb, 256, d, first, h.nb);
        std::vector<float4> shp(h.nb); std::vector<uint32_t> fl(h.nb);
        CK(cudaMemcpyAsync(shp.data(), d.shp + first, h.nb * sizeof(float4), cudaMemcpyDeviceToHost, s));
        CK(cudaMemcpyAsync(fl.data(), d.flags + first, h.nb * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        for (uint32_t k = 0; k < h.nb; ++k) {
            const uint32_t sk = (fl[k] >> F_SHAPE_SHIFT) & 0xFFu;
            const float p[4] = {shp[k].x, shp[k].y, shp[k].z, shp[k].w};
            class_add(w, sk != B2D_SHAPE_NONE ? shape_diameter(sk, p) : 0.0f, (fl[k] & F_KIND_MASK) == 0u);
        }
    }
    if (h.nm) { LAUNCH(k_unpack_manifolds, h.nm, 256, d, h.nm, im, cn.hwm); LAUNCH(k_bump_hwm, 1, 32, d, h.nm); }
    if (h.nh) { LAUNCH(k_unpack_hinges, h.nh, 256, d, d.nhinges, h.nh, ih); d.nhinges += h.nh; }
    if (h.nx) {
        if (2 * (size_t)h.nx > w->stage_floats) { w->error = "b2d_handover_unpack: more exclusions than the staging buffer holds"; return B2D_ERR_CAPACITY; }
        uint2 *loc = (uint2 *)w->stage;
        LAUNCH(k_unpack_exclusions, h.nx, 256, d, ix, h.nx, loc);
        std::vector<uint2> host(h.nx);
        CK(cudaMemcpyAsync(host.data(), loc, h.nx * sizeof(uint2), cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        std::vector<uint64_t> keys; keys.reserve(h.nx);     // both ends are newcomers with fresh local ids: the pairs cannot exist yet
        for (const uint2 &e : host) {
            if (e.x == 0xFFFFFFFFu || e.y == 0xFFFFFFFFu) continue;
            const uint64_t lo = std::min(e.x, e.y), hi = std::max(e.x, e.y);
            keys.push_back((lo << 32) | hi);
        }
        tr.mark("exclusions translated");
        int rc = insert_exclusions(w, keys); if (rc) return rc;
    }
    CK(cudaStreamSynchronize(s));
    tr.mark("done");
    w->labels_stale = true;
    drop_graphs(w);
    if (counts_out) std::memcpy(counts_out, c, sizeof(c));
    return check_device_flags(w);
}

} // extern "C"
