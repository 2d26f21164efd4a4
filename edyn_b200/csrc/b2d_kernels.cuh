// CUDA kernels of the per-step hot path (sm_90a).  One section per reference phase:
//   broadphase   src/edyn/collision/broadphase.cpp:119-195      -> k_bp_*
//   narrowphase  src/edyn/collision/narrowphase.cpp:21-40        -> k_narrowphase
//   islands      src/edyn/simulation/island_manager.cpp:117-247  -> k_cc_*
//   solver       src/edyn/dynamics/solver.cpp:387-468,
//                src/edyn/dynamics/island_solver.cpp:76-111,263-376 -> k_gravity, k_color, k_prepare_*, k_solve,
//                                                                      k_integrate, k_position, k_finalize
// All kernels are grid-stride over device-side counts, so a step needs no host round trip.
#pragma once
#include "b2d_collide.cuh"
#include "b2d_world.cuh"
#include <cooperative_groups.h>

namespace b2d {
namespace cg = cooperative_groups;

#define GRID_STRIDE(i, n) for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x, _s = gridDim.x * blockDim.x; i < (n); i += _s)

B2D_D uint32_t kind_of(uint32_t f) { return f & F_KIND_MASK; }
// "dynamic" on the per-step path = procedural AND awake (every reference view there is exclude_sleeping_disabled);
// a sleeping body behaves like a static one until its island wakes.  is_procedural() is for the island bookkeeping.
B2D_D bool is_dynamic(uint32_t f) { return (f & (F_KIND_MASK | F_SLEEPING)) == 0u; }
B2D_D bool is_procedural(uint32_t f) { return (f & F_KIND_MASK) == 0u; }
B2D_D int shape_of(uint32_t f) { return (int)((f >> F_SHAPE_SHIFT) & 0xFFu); }
B2D_D unsigned long long pair_key(uint32_t a, uint32_t b) {
    return a < b ? ((unsigned long long)a << 32) | b : ((unsigned long long)b << 32) | a;
}
B2D_D uint32_t hash64(unsigned long long k) {
    k ^= k >> 33; k *= 0xff51afd7ed558ccdULL; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ULL; k ^= k >> 33;
    return (uint32_t)k;
}
constexpr unsigned long long EMPTY_KEY = ~0ULL;

// Grid-wide barrier for the persistent (cooperatively launched, hence co-resident) kernels: one release
// atomic + acquire spin per CTA on a monotonic counter that the host zeroes before the launch.
struct GridBarrier {
    unsigned *ctr; unsigned target; unsigned nblocks;
    __device__ __forceinline__ GridBarrier(unsigned *c) : ctr(c), target(0), nblocks(gridDim.x) {}
    __device__ __forceinline__ void sync() {
        __syncthreads();
        if (threadIdx.x == 0) {
            target += nblocks;
            __threadfence();
            atomicAdd(ctr, 1u);
            unsigned v;
            do { asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory"); } while (v < target);
        }
        __syncthreads();
    }
};

B2D_D void hash_insert(unsigned long long *keys, uint32_t *vals, uint32_t size, unsigned long long k, uint32_t v) {
    uint32_t h = hash64(k) & (size - 1);
    for (;;) {
        unsigned long long prev = atomicCAS(&keys[h], EMPTY_KEY, k);
        if (prev == EMPTY_KEY || prev == k) { if (vals) vals[h] = v; return; }
        h = (h + 1) & (size - 1);
    }
}
B2D_D bool hash_find(const unsigned long long *keys, const uint32_t *vals, uint32_t size, unsigned long long k, uint32_t &v) {
    uint32_t h = hash64(k) & (size - 1);
    for (;;) {
        unsigned long long cur = keys[h];
        if (cur == k) { if (vals) v = vals[h]; return true; }
        if (cur == EMPTY_KEY) return false;
        h = (h + 1) & (size - 1);
    }
}

B2D_D box3 body_box(const Dev &d, uint32_t i) { box3 b; b.mn = mk3(d.bbmin[i]); b.mx = mk3(d.bbmax[i]); return b; }
B2D_D m3 load_m3(const float4 *p, uint32_t i) { m3 m; m.r0 = mk3(p[3 * i]); m.r1 = mk3(p[3 * i + 1]); m.r2 = mk3(p[3 * i + 2]); return m; }
B2D_D void store_invIW(const Dev &d, uint32_t i, const m3 &m, float inv_m) {
    d.invIW[3 * i] = f4(m.r0, inv_m); d.invIW[3 * i + 1] = f4(m.r1, 0); d.invIW[3 * i + 2] = f4(m.r2, 0);
}

// ====================================================================== state staging

// Refresh AABB (all shaped bodies) and inertia_world_inv (dynamic) from the current transform:
// util/rigidbody.cpp:75-77,113 at creation; solver.cpp:453-465 after a resync.
__global__ void k_refresh_bodies(Dev d, uint32_t first, uint32_t count) {
    GRID_STRIDE(k, count) {
        uint32_t i = first + k;
        uint32_t f = d.flags[i];
        v3 pos = mk3(d.pos[i]); q4 orn = mkq(d.orn[i]);
        float inv_m = d.pos[i].w;
        if (is_dynamic(f)) store_invIW(d, i, world_inertia(orn, load_m3(d.invI, i)), inv_m);
        else store_invIW(d, i, m3_zero(), 0.0f);
        int sk = shape_of(f);
        if (sk != SH_NONE) { box3 bb = shape_aabb(sk, d.shp[i], pos, orn); d.bbmin[i] = f4(bb.mn, 0); d.bbmax[i] = f4(bb.mx, 0); }
        d.dvw[2 * i] = make_float4(0, 0, 0, 0); d.dvw[2 * i + 1] = make_float4(0, 0, 0, 0);
    }
}

// host float3/float4 packed arrays (staging buffer on device) -> float4 SoA
__global__ void k_unpack_state(Dev d, const float *pos, const float *orn, const float *lv, const float *av, uint32_t n) {
    GRID_STRIDE(i, n) {
        float inv_m = d.pos[i].w;
        d.pos[i] = make_float4(pos[3 * i], pos[3 * i + 1], pos[3 * i + 2], inv_m);
        d.orn[i] = make_float4(orn[4 * i], orn[4 * i + 1], orn[4 * i + 2], orn[4 * i + 3]);
        if (kind_of(d.flags[i]) != 2u) {
            d.linvel[i] = make_float4(lv[3 * i], lv[3 * i + 1], lv[3 * i + 2], 0);
            d.angvel[i] = make_float4(av[3 * i], av[3 * i + 1], av[3 * i + 2], 0);
        }
    }
}
__global__ void k_pack_state(Dev d, float *pos, float *orn, float *lv, float *av, float *bb, float *iw, uint32_t n) {
    GRID_STRIDE(i, n) {
        if (pos) { float4 p = d.pos[i]; pos[3 * i] = p.x; pos[3 * i + 1] = p.y; pos[3 * i + 2] = p.z; }
        if (orn) { float4 q = d.orn[i]; orn[4 * i] = q.x; orn[4 * i + 1] = q.y; orn[4 * i + 2] = q.z; orn[4 * i + 3] = q.w; }
        if (lv) { float4 v = d.linvel[i]; lv[3 * i] = v.x; lv[3 * i + 1] = v.y; lv[3 * i + 2] = v.z; }
        if (av) { float4 v = d.angvel[i]; av[3 * i] = v.x; av[3 * i + 1] = v.y; av[3 * i + 2] = v.z; }
        if (bb) { float4 a = d.bbmin[i], b = d.bbmax[i]; bb[6 * i] = a.x; bb[6 * i + 1] = a.y; bb[6 * i + 2] = a.z; bb[6 * i + 3] = b.x; bb[6 * i + 4] = b.y; bb[6 * i + 5] = b.z; }
        if (iw) { for (int r = 0; r < 3; ++r) { float4 m = d.invIW[3 * i + r]; iw[9 * i + 3 * r] = m.x; iw[9 * i + 3 * r + 1] = m.y; iw[9 * i + 3 * r + 2] = m.z; } }
    }
}

// ====================================================================== broadphase

constexpr float BP_OFFSET = -BREAKING_THRESHOLD;                 // m_aabb_offset, broadphase.hpp:15
constexpr float BP_SEPARATION = -(BREAKING_THRESHOLD * 1.3f);    // -m_separation_threshold, broadphase.hpp:18

// destroy_separated_manifolds (broadphase.cpp:119-134) + rebuild of the pair -> manifold hash
// (contact_manifold_map) from the survivors + dead-slot flags for the free list.
// registry.destroy(body): the node leaves the broadphase trees (broadphase.cpp:54-68) and the entity graph together
// with every edge attached to it (island_manager.cpp:47-66).  Ids are not recycled: the slot turns into a static,
// shapeless body; its manifolds are freed by the next k_bp_separate, its joints are parked on the dead body itself.
__global__ void k_remove_bodies(Dev d, const uint32_t *ids, uint32_t n) {
    GRID_STRIDE(k, n) {
        const uint32_t i = ids[k];
        d.flags[i] = 2u | ((uint32_t)SH_NONE << F_SHAPE_SHIFT) | F_REMOVED;
        d.linvel[i] = make_float4(0, 0, 0, 0); d.angvel[i] = make_float4(0, 0, 0, 0);
        d.dvw[2 * i] = make_float4(0, 0, 0, 0); d.dvw[2 * i + 1] = make_float4(0, 0, 0, 0);
        d.pos[i].w = 0.0f;
        store_invIW(d, i, m3_zero(), 0.0f);
    }
}
__global__ void k_remove_hinges(Dev d) {
    GRID_STRIDE(h, d.nhinges) {
        const uint2 p = d.hpair[h];
        const bool ra = d.flags[p.x] & F_REMOVED, rb = d.flags[p.y] & F_REMOVED;
        if (ra || rb) { const uint32_t dead = ra ? p.x : p.y; d.hpair[h] = make_uint2(dead, dead); d.hcolor[h] = COLOR_NONE; }
    }
}
__global__ void k_bp_separate(Dev d) {
    const uint32_t hwm = d.cnt->hwm;
    GRID_STRIDE(m, d.NM) {
        uint32_t flag = 0;
        if (m < hwm) {
            uint32_t st = d.mstate[m];
            if (st & MS_ALIVE) {
                uint2 p = d.mpair[m];
                // a destroyed body takes its graph edges with it (island_manager.cpp:47-66)
                if (((d.flags[p.x] | d.flags[p.y]) & F_REMOVED) || !intersect(inset(body_box(d, p.x), BP_SEPARATION), body_box(d, p.y))) {
                    d.mstate[m] = COLOR_NONE << MS_COLOR_SHIFT;      // clear_contact_manifold + destroy
                    d.cnt->graph_changed = 1u;
                    flag = 1;
                } else {
                    hash_insert(d.mhash_key, d.mhash_val, d.mhash_size, pair_key(p.x, p.y), m);
                }
            } else flag = 1;
        }
        d.free_flag[m] = flag;
    }
}
__global__ void k_bp_free_list(Dev d) {
    GRID_STRIDE(m, d.NM) {
        if (d.free_flag[m]) d.free_list[d.free_rank[m]] = m;
        if (m == d.NM - 1) d.cnt->nfree = d.free_rank[m] + d.free_flag[m];
    }
}

// Cell key: the three cell coordinates relative to d.cell_org, packed into d.cell_bits[0..2] bits each (radix sort
// passes are paid per key byte, so the host sizes the fields to the extent the world had when the step was captured).
// Cells beyond the range share the boundary key, which only makes the candidate lists there longer: every pair still
// goes through the exact AABB tests.  Neighbour offsets that clamp to the same field are the same cells: clamping is
// monotone, so they are adjacent, and the search skips an offset whose field repeats the previous offset's on some axis
// (each cell is walked once per query body).  All-ones is reserved for "no cell", so x stops one short of its field's maximum.
struct CellFields { uint32_t x, y, z; };
B2D_D uint32_t cell_field(const Dev &d, int k, int c) {
    return (uint32_t)min(max(c - d.cell_org[k], 0), (1 << d.cell_bits[k]) - (k == 0 ? 2 : 1));
}
B2D_D CellFields cell_fields(const Dev &d, int cx, int cy, int cz) {
    return CellFields{cell_field(d, 0, cx), cell_field(d, 1, cy), cell_field(d, 2, cz)};
}
B2D_D unsigned long long cell_key(const Dev &d, CellFields f) {
    return ((unsigned long long)f.x << (d.cell_bits[1] + d.cell_bits[2])) | ((unsigned long long)f.y << d.cell_bits[2]) | f.z;
}
B2D_D unsigned long long cell_key_of(const Dev &d, int cx, int cy, int cz) { return cell_key(d, cell_fields(d, cx, cy, cz)); }
// The box of key fields occupied this step (k_bp_cells): a cell outside it is empty, so its hash probe is skipped.
struct CellBox { uint32_t lo[3], hi[3]; };
B2D_D CellBox load_cell_box(const Dev &d) {
    CellBox b;
    #pragma unroll
    for (int k = 0; k < 3; ++k) { b.lo[k] = d.cell_box[k]; b.hi[k] = ~d.cell_box[3 + k]; }
    return b;
}
B2D_D bool in_cell_box(const CellBox &b, CellFields f) {
    return f.x >= b.lo[0] && f.x <= b.hi[0] && f.y >= b.lo[1] && f.y <= b.hi[1] && f.z >= b.lo[2] && f.z <= b.hi[2];
}
B2D_D void cell_of(const Dev &d, float4 a, float4 b, int &cx, int &cy, int &cz) {
    cx = (int)floorf((a.x + b.x) * 0.5f * d.inv_cell);
    cy = (int)floorf((a.y + b.y) * 0.5f * d.inv_cell);
    cz = (int)floorf((a.z + b.z) * 0.5f * d.inv_cell);
}
B2D_D void cell_of(const Dev &d, uint32_t i, int &cx, int &cy, int &cz) { cell_of(d, d.bbmin[i], d.bbmax[i], cx, cy, cz); }

// Cell key per body.  Shapeless and "large" bodies get the all-ones key and sort to the end.  The broadphase writes
// d.cellkey / d.cellbody and the occupied box of key fields (box: min field, then min of the complemented field, both
// preset to all-ones); the raycast index (k_ray_*) its own arrays and no box.
__global__ void k_bp_cells(Dev d, unsigned long long *cellkey, uint32_t *cellbody, uint32_t *box) {
    uint32_t m[6] = {~0u, ~0u, ~0u, ~0u, ~0u, ~0u};
    GRID_STRIDE(i, d.nbodies) {
        uint32_t f = d.flags[i];
        unsigned long long key = EMPTY_KEY;
        if (shape_of(f) != SH_NONE && !(f & F_LARGE)) {
            int cx, cy, cz; cell_of(d, i, cx, cy, cz);
            const CellFields c = cell_fields(d, cx, cy, cz);
            key = cell_key(d, c);
            m[0] = min(m[0], c.x); m[1] = min(m[1], c.y); m[2] = min(m[2], c.z);
            m[3] = min(m[3], ~c.x); m[4] = min(m[4], ~c.y); m[5] = min(m[5], ~c.z);
        }
        cellkey[i] = key; cellbody[i] = i;
    }
    if (!box) return;
    __shared__ uint32_t sm[6];
    if (threadIdx.x < 6) sm[threadIdx.x] = ~0u;
    __syncthreads();
    #pragma unroll
    for (int k = 0; k < 6; ++k) {
        m[k] = __reduce_min_sync(0xffffffffu, m[k]);
        if ((threadIdx.x & 31) == 0) atomicMin(&sm[k], m[k]);
    }
    __syncthreads();
    if (threadIdx.x < 6 && sm[threadIdx.x] != ~0u) atomicMin(&box[threadIdx.x], sm[threadIdx.x]);
}
// Cells occupied by the bodies that go into the grid (host: sizes the key fields, b2d_api.cu measure_cells)
__global__ void k_cell_extent(Dev d, int *out6) {
    int mn[3] = {0x7FFFFFFF, 0x7FFFFFFF, 0x7FFFFFFF}, mx[3] = {-0x7FFFFFFF, -0x7FFFFFFF, -0x7FFFFFFF};
    GRID_STRIDE(i, d.nbodies) {
        const uint32_t f = d.flags[i];
        if (shape_of(f) == SH_NONE || (f & F_LARGE)) continue;
        int c[3]; cell_of(d, i, c[0], c[1], c[2]);
        #pragma unroll
        for (int k = 0; k < 3; ++k) { mn[k] = min(mn[k], c[k]); mx[k] = max(mx[k], c[k]); }
    }
    #pragma unroll
    for (int k = 0; k < 3; ++k) {
        mn[k] = __reduce_min_sync(0xffffffffu, mn[k]); mx[k] = __reduce_max_sync(0xffffffffu, mx[k]);
        if ((threadIdx.x & 31) == 0 && mn[k] <= mx[k]) { atomicMin(&out6[k], mn[k]); atomicMax(&out6[3 + k], mx[k]); }
    }
}
// The body a manifold is filed under (sort key, tile, spatial rank): a dynamic one whenever it has one, the non-large one
// of two dynamic bodies (its spatial rank is meaningful), a non-dynamic one only when neither is dynamic.  This is the
// root rule of the island census (k_color_list) and of the hinges' keys (k_color_keys): every constraint of a tiled
// island sorts into its tile's range, so k_island_tiles sees all of a tiled body's constraints and the dataflow path none
// of them.
B2D_D uint32_t key_body(const Dev &d, uint2 pr) {
    const uint32_t fa = d.flags[pr.x], fb = d.flags[pr.y];
    return (is_dynamic(fa) && (!(fa & F_LARGE) || !is_dynamic(fb))) ? pr.x : pr.y;
}
// spatial part of a dataflow manifold's sort key (k_color_keys): the key body's rank in the cell order, 14 bits
B2D_D uint32_t df_spatial(const Dev &d, uint32_t rank) { return (uint32_t)(((unsigned long long)rank << KEY_DF_SPATIAL_BITS) / d.nbodies); }
// First sorted index of every occupied cell -> hash table, and every body's candidate record in the sorted order (what
// bp_candidate reads about it), so the neighbourhood search walks records instead of gathering by body id.  A body that
// is not in an island tile and whose spatial rank moved would change a dataflow sort key: the island rebuild has to run.
__global__ void k_bp_cell_starts(Dev d) {
    GRID_STRIDE(i, d.nbodies) {
        // the gathers first: they are independent of each other and of the hash insert's atomics
        const uint32_t b = d.cellbody_s[i];
        const float4 mn = d.bbmin[b], mx = d.bbmax[b];
        d.bprec_min[i] = make_float4(mn.x, mn.y, mn.z, __uint_as_float(b));
        d.bprec_max[i] = make_float4(mx.x, mx.y, mx.z, __uint_as_float(d.flags[b]));
        unsigned long long k = d.cellkey_s[i];
        if (k != EMPTY_KEY && (i == 0 || d.cellkey_s[i - 1] != k)) hash_insert(d.chash_key, d.chash_val, d.chash_size, k, i);
        if (df_spatial(d, d.brank[b]) != df_spatial(d, i) && d.btile[b] == TILE_NONE) d.cnt->graph_changed = 1u;
        d.brank[b] = i;
    }
}

// should_collide_default, collision/should_collide.cpp:23-57 (exclusion list kept as a pair hash set)
B2D_D bool should_collide(const Dev &d, uint32_t a, uint32_t fa, uint32_t b, uint32_t fb) {
    bool ha = fa & F_FILTER, hb = fb & F_FILTER;
    if (ha && hb) {
        if ((d.group[a] & d.fmask[b]) == 0ULL || (d.group[b] & d.fmask[a]) == 0ULL) return false;
    } else if (ha || hb) {
        uint32_t f = ha ? a : b;
        if (d.group[f] == 0ULL || d.fmask[f] == 0ULL) return false;
    }
    if (d.xhash_size) { uint32_t v; if (hash_find(d.xhash_key, nullptr, d.xhash_size, pair_key(a, b), v)) return false; }
    return true;
}

// One query body A against one candidate j.  The reference creates a manifold when EITHER body's query
// (its AABB inflated by 0.02) hits the other's AABB, whichever is iterated first (broadphase.cpp:183-194,
// :136-155).  Each unordered pair is evaluated by exactly one thread: the one of the higher-id procedural
// body (views are assumed to iterate newest-first, SURVEY.md appendix A.11), which therefore becomes body[0].
// (j, fj, bbj) are the candidate's id, flags and AABB, from its cell-ordered record (bp_candidate_rec) or gathered by
// id (bp_candidate_id).
B2D_D void bp_candidate(const Dev &d, uint32_t A, uint32_t fA, const box3 &bbA, const box3 &qA, uint32_t j, uint32_t fj,
                        const box3 &bbj, uint32_t &count, uint2 *out) {
    if (j == A) return;
    if (shape_of(fj) == SH_NONE) return;
    bool pj = is_dynamic(fj);
    if (pj && j > A) return;
    uint32_t first = A, second = j;
    if (pj) {
        bool t1 = intersect(qA, bbj);
        if (!t1) {
            if (!intersect(inset(bbj, BP_OFFSET), bbA)) return;
            first = j; second = A;
        }
    } else if (!intersect(qA, bbj)) return;
    if (!should_collide(d, A, fA, j, fj)) return;
    uint32_t v;
    if (hash_find(d.mhash_key, d.mhash_val, d.mhash_size, pair_key(A, j), v)) return;
    if (out) out[count] = make_uint2(first, second);
    ++count;
}
B2D_D void bp_candidate_id(const Dev &d, uint32_t A, uint32_t fA, const box3 &bbA, const box3 &qA, uint32_t j,
                           uint32_t &count, uint2 *out) {
    bp_candidate(d, A, fA, bbA, qA, j, d.flags[j], body_box(d, j), count, out);
}
B2D_D box3 rec_box(float4 mn, float4 mx) { box3 b; b.mn = mk3(mn); b.mx = mk3(mx); return b; }
B2D_D void bp_candidate_rec(const Dev &d, uint32_t A, uint32_t fA, const box3 &bbA, const box3 &qA, uint32_t k,
                            uint32_t &count, uint2 *out) {
    const float4 mn = d.bprec_min[k], mx = d.bprec_max[k];
    bp_candidate(d, A, fA, bbA, qA, __float_as_uint(mn.w), __float_as_uint(mx.w), rec_box(mn, mx), count, out);
}

// One column of the 27-cell neighbourhood: the cells (x, y, cz - 1 .. cz + 1).  z is the key's low field, so cells with
// consecutive keys are one run of the sorted records, and one walk from the run's first occupied cell visits them in the
// order of a probe and a walk per cell.  Where cell_key_of clamps z (outside the extent measured at capture), two or
// three offsets share a key; only the first of them is probed, so the cell is walked once and each pair found once.
struct BpColumn { unsigned long long key[3]; uint32_t start[3]; bool occ[3]; };
B2D_D BpColumn bp_column_find(const Dev &d, const CellBox &box, int x, int y, int cz) {
    BpColumn c;
    #pragma unroll
    for (int z = 0; z < 3; ++z) {
        const CellFields f = cell_fields(d, x, y, cz + z - 1);
        c.key[z] = cell_key(d, f);
        c.occ[z] = (z == 0 || c.key[z] != c.key[z - 1]) && in_cell_box(box, f) && hash_find(d.chash_key, d.chash_val, d.chash_size, c.key[z], c.start[z]);
    }
    return c;
}
B2D_D void bp_column_walk(const Dev &d, const BpColumn &c, uint32_t A, uint32_t fA, const box3 &bbA, const box3 &qA,
                          uint32_t &count, uint2 *out) {
    bool found = false; uint32_t k = 0;
    #pragma unroll
    for (int z = 0; z < 3; ++z) {
        if (!found && c.occ[z]) { found = true; k = c.start[z]; }
        if (z == 2 || c.key[z + 1] != c.key[z] + 1) {             // the run ends at cell z
            if (found) for (; k < d.nbodies && d.cellkey_s[k] <= c.key[z]; ++k) bp_candidate_rec(d, A, fA, bbA, qA, k, count, out);
            found = false;
        }
    }
}

template<bool FILL>
__global__ void k_bp_pairs(Dev d) {
    GRID_STRIDE(t, d.nbodies) {
        // threads walk the bodies in cell order: a warp's queries hit the same cells and candidate records (output
        // slots are still indexed by body id, so the pair order does not change)
        const float4 rmn = d.bprec_min[t], rmx = d.bprec_max[t];
        const uint32_t A = __float_as_uint(rmn.w), fA = __float_as_uint(rmx.w);
        uint32_t count = 0;
        uint2 *out = nullptr;
        if (FILL) {
            if (d.newcount[A] == 0) continue;
            // newpairs holds max_manifolds entries: a body whose range would run past it (and therefore every body behind
            // it in the scan) is dropped, the append below stops in front of the first hole
            if ((unsigned long long)d.newoff[A] + d.newcount[A] > d.NM) { atomicOr(&d.cnt->err, ERR_MANIFOLD_CAPACITY); continue; }
            out = d.newpairs + d.newoff[A];
        }
        if (is_dynamic(fA) && shape_of(fA) != SH_NONE) {
            const box3 bbA = rec_box(rmn, rmx);
            const box3 qA = inset(bbA, BP_OFFSET);
            if (!(fA & F_LARGE)) {
                int cx, cy, cz; cell_of(d, rmn, rmx, cx, cy, cz);
                const CellBox box = load_cell_box(d);
                for (int dx = -1; dx <= 1; ++dx) {
                    if (dx > -1 && cell_field(d, 0, cx + dx) == cell_field(d, 0, cx + dx - 1)) continue;      // clamped: same cells
                    for (int dy = -1; dy <= 1; ++dy) {
                        if (dy > -1 && cell_field(d, 1, cy + dy) == cell_field(d, 1, cy + dy - 1)) continue;
                        bp_column_walk(d, bp_column_find(d, box, cx + dx, cy + dy, cz), A, fA, bbA, qA, count, out);
                    }
                }
            } else {
                for (uint32_t j = 0; j < d.nbodies; ++j) if (!(d.flags[j] & F_LARGE)) bp_candidate_id(d, A, fA, bbA, qA, j, count, out);
            }
            for (uint32_t k = 0; k < d.nlarge; ++k) bp_candidate_id(d, A, fA, bbA, qA, d.large_list[k], count, out);
        }
        if (!FILL) d.newcount[A] = count;
    }
}
// The same search with one WARP per query body: lane c < 27 takes cell c of the neighbourhood (in the loop order of
// the thread-per-body kernel: its column walks visit the same cells in the same order; a lane whose cell repeats an
// earlier lane's clamped cell stays idle), lane 27 the large list; a large
// query body splits the brute-force list over lanes 0..26.  A warp prefix sum of the lane counts puts the pairs in
// exactly the order the serial walk produces.  27 probes and cell walks in flight per body: the search is latency-bound
// at small body counts, where a lane per column (three cells walked one after the other) was slower (DESIGN.md §2).
template<bool FILL>
// (launch bounds: the repeat test below costs registers; bounded, both passes keep at least the residency they had without it)
__global__ void __launch_bounds__(256, FILL ? 5 : 8) k_bp_pairs_warp(Dev d) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t wid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t t = wid; t < d.nbodies; t += nw) {
        const float4 rmn = d.bprec_min[t], rmx = d.bprec_max[t];
        const uint32_t A = __float_as_uint(rmn.w), fA = __float_as_uint(rmx.w);
        uint2 *out = nullptr;
        if (FILL) {
            if (d.newcount[A] == 0) continue;
            if ((unsigned long long)d.newoff[A] + d.newcount[A] > d.NM) { if (lane == 0) atomicOr(&d.cnt->err, ERR_MANIFOLD_CAPACITY); continue; }
            out = d.newpairs + d.newoff[A];
        }
        uint32_t total = 0;
        if (is_dynamic(fA) && shape_of(fA) != SH_NONE) {
            const box3 bbA = rec_box(rmn, rmx);
            const box3 qA = inset(bbA, BP_OFFSET);
            // this lane's share of the candidates, walked once to count and (FILL) once more to write
            uint32_t start = 0, end = 0; unsigned long long key = EMPTY_KEY; int mode = 0;      // 0 nothing, 1 one cell, 2 a range of body ids, 3 the large list
            if (!(fA & F_LARGE)) {
                if (lane < 27u) {
                    int cx, cy, cz; cell_of(d, rmn, rmx, cx, cy, cz);
                    const int ox = (int)(lane / 9u), oy = (int)((lane / 3u) % 3u), oz = (int)(lane % 3u);
                    const CellFields f = cell_fields(d, cx + ox - 1, cy + oy - 1, cz + oz - 1);
                    key = cell_key(d, f);
                    // a lane whose field repeats the previous offset's on some axis has the same cell as an earlier lane
                    const bool repeat = (ox && f.x == cell_field(d, 0, cx + ox - 2)) || (oy && f.y == cell_field(d, 1, cy + oy - 2)) ||
                                        (oz && f.z == cell_field(d, 2, cz + oz - 2));
                    if (!repeat && in_cell_box(load_cell_box(d), f) && hash_find(d.chash_key, d.chash_val, d.chash_size, key, start)) mode = 1;
                }
            } else if (lane < 27u) {
                const uint32_t chunk = (d.nbodies + 26u) / 27u;
                start = min(lane * chunk, d.nbodies); end = min(start + chunk, d.nbodies); mode = 2;
            }
            if (lane == 27u) mode = 3;
            auto walk = [&](uint2 *o) {
                uint32_t c = 0;
                if (mode == 1) { for (uint32_t k = start; k < d.nbodies && d.cellkey_s[k] == key; ++k) bp_candidate_rec(d, A, fA, bbA, qA, k, c, o); }
                else if (mode == 2) { for (uint32_t j = start; j < end; ++j) if (!(d.flags[j] & F_LARGE)) bp_candidate_id(d, A, fA, bbA, qA, j, c, o); }
                else if (mode == 3) { for (uint32_t k = 0; k < d.nlarge; ++k) bp_candidate_id(d, A, fA, bbA, qA, d.large_list[k], c, o); }
                return c;
            };
            const uint32_t mine = walk(nullptr);
            uint32_t incl = mine;
            #pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= (uint32_t)o) incl += v; }
            total = __shfl_sync(0xffffffffu, incl, 31);
            if (FILL && mine) walk(out + (incl - mine));
        }
        if (!FILL && lane == 0) d.newcount[A] = total;
    }
}
// Number of new pairs this step.  newpairs holds max_manifolds entries: a body whose range would run past it (and
// therefore every body behind it in the scan) is dropped by the fill pass, so the usable prefix ends where the first
// such range starts (found by bisection on the monotone prefix sums; only on overflow).
B2D_D uint32_t bp_nnew(const Dev &d) {
    const uint32_t n = d.nbodies;
    if (!n) return 0;
    const unsigned long long total = (unsigned long long)d.newoff[n - 1] + d.newcount[n - 1];
    if (total <= d.NM) return (uint32_t)total;
    uint32_t lo = 0, hi = n - 1;                       // first body whose range ends beyond the buffer
    while (lo < hi) { const uint32_t mid = (lo + hi) / 2; if ((unsigned long long)d.newoff[mid] + d.newcount[mid] > d.NM) hi = mid; else lo = mid + 1; }
    return d.newoff[lo];
}
// make_contact_manifold (util/constraint_util.cpp:67-102): slots come from the free list first.
__global__ void k_bp_append(Dev d) {
    const uint32_t nnew = bp_nnew(d), nfree = d.cnt->nfree, hwm = d.cnt->hwm;
    GRID_STRIDE(k, nnew) {
        uint32_t slot = k < nfree ? d.free_list[k] : hwm + (k - nfree);
        if (slot >= d.NM) { atomicOr(&d.cnt->err, ERR_MANIFOLD_CAPACITY); continue; }
        d.mpair[slot] = d.newpairs[k];
        d.mstate[slot] = MS_ALIVE | (COLOR_NONE << MS_COLOR_SHIFT);
    }
}
__global__ void k_bp_finish(Dev d) {
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        Counters &c = *d.cnt;
        c.nnew = bp_nnew(d);
        if (c.nnew > c.nfree) c.hwm = min(d.NM, c.hwm + (c.nnew - c.nfree));
        if (c.nnew) c.graph_changed = 1u;
    }
}

// ====================================================================== narrowphase

B2D_D unsigned lbits(float4 pl) { return __float_as_uint(pl.w); }

// collision_util.cpp:233-255
B2D_D int find_nearest_contact(v3 cpA, v3 cpB, const CResult &res) {
    float shortest = CACHING_THRESHOLD * CACHING_THRESHOLD;
    int nearest = res.num;
    #pragma unroll 1
    for (int i = 0; i < res.num; ++i) {
        float dA = length_sqr(res.pt[i].pivotA - cpA);
        float dB = length_sqr(res.pt[i].pivotB - cpB);
        if (dA < shortest) { shortest = dA; nearest = i; }
        if (dB < shortest) { shortest = dB; nearest = i; }
    }
    return nearest;
}
// collision_util.cpp:257-280 (uses result.pivotA for either body, like the reference)
B2D_D int find_nearest_contact_rolling(const CResult &res, v3 cp_pivot, v3 origin, q4 orn, v3 angvel, float dt) {
    int nearest = res.num;
    q4 prev_orn = integrate(orn, angvel, -dt);
    v3 prev_pivot = to_world(cp_pivot, origin, prev_orn);
    float shortest = CACHING_THRESHOLD * CACHING_THRESHOLD;
    for (int i = 0; i < res.num; ++i) {
        v3 pA = to_world(res.pt[i].pivotA, origin, orn);
        float ds = distance_sqr(pA, prev_pivot);
        if (ds < shortest) { shortest = ds; nearest = i; }
    }
    return nearest;
}

// One contact point in registers, without its warm-start impulse: pI is only touched where a point changes slots or
// is created (np_merge), so a point that stays where it is keeps its impulse without a load or a store.
struct MPoint {
    v3 pivotA, pivotB, normal, local_normal;
    float distance, friction, restitution;
    unsigned att, lifetime;
};
B2D_D void load_point(const Dev &d, uint32_t m, int s, MPoint &p) {
    size_t i = (size_t)s * d.NM + m;
    float4 a = d.pA[i], b = d.pB[i], n = d.pN[i], l = d.pL[i];
    p.pivotA = mk3(a); p.distance = a.w; p.pivotB = mk3(b); p.friction = b.w; p.normal = mk3(n); p.restitution = n.w;
    p.local_normal = mk3(l); unsigned u = __float_as_uint(l.w); p.att = u & 3u; p.lifetime = u >> 2;
}
B2D_D void store_point(const Dev &d, uint32_t m, int s, const MPoint &p) {
    size_t i = (size_t)s * d.NM + m;
    d.pA[i] = f4(p.pivotA, p.distance); d.pB[i] = f4(p.pivotB, p.friction); d.pN[i] = f4(p.normal, p.restitution);
    d.pL[i] = f4(p.local_normal, __uint_as_float((p.att & 3u) | (p.lifetime << 2)));
}
// merge_point, collision_util.cpp:205-231
B2D_D void merge_point(const CPoint &rp, MPoint &cp, q4 ornA, q4 ornB) {
    cp.pivotA = rp.pivotA; cp.pivotB = rp.pivotB; cp.normal = rp.normal; cp.distance = rp.distance; cp.att = rp.att;
    if (rp.att != ATT_NONE) cp.local_normal = rotate(conjugate(rp.att == ATT_A ? ornA : ornB), rp.normal);
    else cp.local_normal = mk3(0, 0, 0);
}
// create_contact_point, collision_util.cpp:319-395; mixing dynamics/material_mixing.hpp:12-18
B2D_D MPoint create_point(const CPoint &rp, q4 ornA, q4 ornB, float2 matA, float2 matB) {
    MPoint cp;
    cp.pivotA = rp.pivotA; cp.pivotB = rp.pivotB; cp.normal = rp.normal; cp.att = rp.att; cp.distance = rp.distance;
    if (rp.att != ATT_NONE) cp.local_normal = rotate(conjugate(rp.att == ATT_A ? ornA : ornB), rp.normal);
    else cp.local_normal = mk3(0, 0, 0);
    cp.friction = sqrtf(matA.x * matB.x);
    cp.restitution = fminf(matA.y, matB.y);
    cp.lifetime = 0;
    return cp;
}
B2D_D int nth_set_bit(unsigned mask, int n) {          // position of the n-th (from 0) set bit of mask
    for (int k = 0; k < n; ++k) mask &= mask - 1u;
    return __ffs(mask) - 1;
}

// Narrowphase in three steps:
//   k_np_keys     pair-type key per manifold slot + histogram, k_np_scatter the counting sort by type, so that
//   k_np_collide  runs the collision of every awake manifold over the sorted list, where a warp's lanes run the same
//                 collide() overload (no divergence between sphere/box/capsule code paths but at the range edges),
//                 and merges the result, still in registers, into the manifold's points (np_merge).
//                 k_np_collide<5> (box-box) and <9> (capsule-box) take a launch each, k_np_collide_light the rest.
__global__ void k_np_keys(Dev d) {
    __shared__ uint32_t s_hist[16];
    if (threadIdx.x < 16) s_hist[threadIdx.x] = 0;
    __syncthreads();
    const uint32_t hwm = d.cnt->hwm;
    GRID_STRIDE(m, hwm) {
        uint32_t key = 0xFF;
        if (d.mstate[m] & MS_ALIVE) {
            uint2 pr = d.mpair[m];
            if (is_dynamic(d.flags[pr.x]) || is_dynamic(d.flags[pr.y])) {      // else: sleeping manifold (narrowphase.cpp:31)
                int ka = shape_of(d.flags[pr.x]), kb = shape_of(d.flags[pr.y]);
                int fn = pair_fn(ka, kb);
                if (!fn) fn = pair_fn(kb, ka);
                key = (uint32_t)fn;
            }
        }
        d.ckey[m] = key;
        if (key != 0xFF) atomicAdd(&s_hist[key & 15u], 1u);       // histogram of the pair types, per CTA first
    }
    __syncthreads();
    if (threadIdx.x < 16 && s_hist[threadIdx.x]) atomicAdd(&d.cnt->npcount[threadIdx.x], s_hist[threadIdx.x]);
}
// Counting sort by pair type: manifold slots of one type become a contiguous range of npidx.  Every CTA takes windows
// of 256 consecutive slots, keeps their order inside a type (manifold slots are spatially coherent, the detect kernels
// gather body data through them) and claims the window's share of each range with one atomic per type; which window
// comes first is first come first served -- it only decides which thread runs which manifold.
__global__ void __launch_bounds__(256) k_np_scatter(Dev d) {
    __shared__ uint32_t s_off[16], s_base[16], s_wcount[8][16];
    Counters &c = *d.cnt;
    if (threadIdx.x == 0) {
        uint32_t acc = 0;
        for (int k = 0; k < 16; ++k) { s_off[k] = acc; acc += c.npcount[k]; }
        if (blockIdx.x == 0) for (int k = 0; k < 16; ++k) c.npoff[k] = s_off[k];
    }
    const uint32_t hwm = c.hwm, lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    for (uint32_t w0 = blockIdx.x * 256u; w0 < hwm; w0 += gridDim.x * 256u) {
        if (threadIdx.x < 128) s_wcount[threadIdx.x >> 4][threadIdx.x & 15u] = 0;
        __syncthreads();
        const uint32_t m = w0 + threadIdx.x;
        const uint32_t key = m < hwm ? d.ckey[m] : 0xFFu;
        const uint32_t grp = __match_any_sync(0xffffffffu, key);
        const uint32_t rank = __popc(grp & ((1u << lane) - 1u));
        if (key != 0xFFu && rank == 0) s_wcount[warp][key & 15u] = __popc(grp);
        __syncthreads();
        if (threadIdx.x < 16) {          // exclusive prefix over the warps, then the window's claim on the type's range
            uint32_t acc = 0;
            for (int w = 0; w < 8; ++w) { const uint32_t n = s_wcount[w][threadIdx.x]; s_wcount[w][threadIdx.x] = acc; acc += n; }
            s_base[threadIdx.x] = acc ? atomicAdd(&c.npcursor[threadIdx.x], acc) : 0u;
        }
        __syncthreads();
        if (key != 0xFFu) d.npidx[s_off[key & 15u] + s_base[key & 15u] + s_wcount[warp][key & 15u] + rank] = m;
        __syncthreads();
    }
}

// update_contact_distances (collision_util.cpp:28-45) + process_collision (collision_util.hpp:105-276, sequential flavour
// of narrowphase.hpp:62-84) of alive, awake manifold m with this step's collision result res.  The manifold's state and
// pair and the bodies' flags and poses are read here, after the collision, rather than held in registers across it.
//
// No per-point array: the state of the (at most 4) points is kept in bit fields, the points themselves in their slots
// in HBM, so nothing here is indexed at run time but res, and the merge adds nothing to the local frame.  Each persisted
// point is updated in its own slot as soon as it is processed.  When every point stays and every result point merged
// into one -- the settled case -- that is all.  Otherwise np_rearrange moves the points into the reference's order.
//
// np_rearrange: the rest of process_collision once the persisted points are merged and stored in place.  `keep` says
// which slots hold a point that stays, `merged` which result points a persisted point took.  Inserts the other result
// points and writes the final list, newest first and capped at 4, moving impulses with the points; returns its length.
B2D_D int np_rearrange(const Dev &d, uint32_t m, uint2 pr, const CResult &res, unsigned keep, unsigned merged) {
    const int num = __popc(keep);       // the persisted list after the removals: its point j sits in slot nth_set_bit(keep, j)
    // ---- insertion.  L is the persisted list with the result points written over it: slot j of L is persisted point
    //      j while type j is INS_NONE, else result point lsrc j (2 bits per slot in `type` and `lsrc`)
    int num_points = num;
    unsigned type = 0u, lsrc = 0u;
    if (merged != (1u << res.num) - 1u) {
        if (num_points == 0) { num_points = 1; type = INS_APPEND; merged |= 1u; }
        auto piv = [&](int j, bool B) -> v3 {           // pivot A or B of slot j of L
            if (j >= num_points) return mk3(0, 0, 0);   // not read by insertion_index
            if (type >> 2 * j & 3u) { const CPoint &q = res.pt[lsrc >> 2 * j & 3u]; return B ? q.pivotB : q.pivotA; }
            const size_t i = (size_t)nth_set_bit(keep, j) * d.NM + m;
            return mk3(B ? d.pB[i] : d.pA[i]);
        };
        #pragma unroll 1
        for (int k = 0; k < res.num; ++k) {
            if (merged >> k & 1u) continue;
            int idx, t = INS_NONE;
            #pragma unroll 1
            for (int B = 0; B < 2 && t == INS_NONE; ++B)          // pivots A, then pivots B if A found no place
                t = insertion_index(piv(0, B), piv(1, B), piv(2, B), piv(3, B), num_points, B ? res.pt[k].pivotB : res.pt[k].pivotA, idx);
            if (t != INS_NONE && idx >= 0 && idx < 4) {
                type = (type & ~(3u << 2 * idx)) | (unsigned)t << 2 * idx;
                lsrc = (lsrc & ~(3u << 2 * idx)) | (unsigned)k << 2 * idx;
            }
        }
    }
    // ---- the slots of L that become new points (appended, similar to no persisted point, or replacing one), and the
    //      persisted points that stay alive
    unsigned created = 0u, alive = (1u << num) - 1u;
    for (int j = 0; j < num_points; ++j) {
        const unsigned t = type >> 2 * j & 3u;
        if (t == INS_APPEND || t == INS_REPLACE || (t == INS_SIMILAR && j >= num)) created |= 1u << j;
        if (t == INS_REPLACE && j < num) alive &= ~(1u << j);
    }
    const int n_created = __popc(created);
    // ---- the list: the created points newest first, then the alive persisted points in order, at most 4.  Persisted
    //      point j moves from slot s to slot n_created + (alive points before it); both grow with j, so the points that
    //      move up go first, last point first, then the rest in order, and no point is overwritten before it moved
    auto place = [&](int j, bool up) {
        if (!(alive >> j & 1u)) return;
        const int s = nth_set_bit(keep, j), dst = n_created + __popc(alive & ((1u << j) - 1u));
        const bool similar = (type >> 2 * j & 3u) == INS_SIMILAR;
        if (dst >= MAX_CONTACTS || (dst > s) != up || (dst == s && !similar)) return;
        MPoint cp;
        load_point(d, m, s, cp);
        if (similar) merge_point(res.pt[lsrc >> 2 * j & 3u], cp, mkq(d.orn[pr.x]), mkq(d.orn[pr.y]));
        store_point(d, m, dst, cp);
        if (dst != s) d.pI[(size_t)dst * d.NM + m] = f4(mk3(d.pI[(size_t)s * d.NM + m]), 0);
    };
    #pragma unroll 1
    for (int j = num - 1; j >= 0; --j) place(j, true);
    #pragma unroll 1
    for (int j = 0; j < num; ++j) place(j, false);
    if (created) {
        const float2 matA = d.mat[pr.x], matB = d.mat[pr.y];
        const q4 ornA = mkq(d.orn[pr.x]), ornB = mkq(d.orn[pr.y]);
        int dst = n_created;
        #pragma unroll 1
        for (int j = 0; j < num_points; ++j) {
            if (!(created >> j & 1u)) continue;
            store_point(d, m, --dst, create_point(res.pt[lsrc >> 2 * j & 3u], ornA, ornB, matA, matB));
            d.pI[(size_t)dst * d.NM + m] = make_float4(0, 0, 0, 0);
        }
    }
    return min(MAX_CONTACTS, n_created + __popc(alive));
}
B2D_D void np_merge(const Dev &d, uint32_t m, const CResult &res) {
    const uint32_t st = d.mstate[m];
    const uint2 pr = d.mpair[m];
    const int num0 = (int)(st & MS_NPTS_MASK);
    if (num0 == 0 && res.num == 0) return;
    const uint32_t a = pr.x, b = pr.y, fa = d.flags[a], fb = d.flags[b];
    const v3 posA = mk3(d.pos[a]), posB = mk3(d.pos[b]);
    const q4 ornA = mkq(d.orn[a]), ornB = mkq(d.orn[b]);
    // ---- merge with persisted points, in their order.  The reference erases a removed point from its list, which
    //      shifts the later ones down; here it clears the point's bit in `keep`, and np_rearrange closes the gap.
    unsigned merged = 0u, keep = 0u;        // bit k: res.pt[k] was merged into a point; bit s: the point of slot s stays
    const bool rollA = fa & F_ROLLING, rollB = fb & F_ROLLING;
    #pragma unroll 1
    for (int s = 0; s < num0; ++s) {
        MPoint cp;
        load_point(d, m, s, cp);
        ++cp.lifetime;
        int nearest = find_nearest_contact(cp.pivotA, cp.pivotB, res);
        if (nearest == res.num && rollA) nearest = find_nearest_contact_rolling(res, cp.pivotA, posA, ornA, mk3(d.angvel[a]), d.dt);
        if (nearest == res.num && rollB) nearest = find_nearest_contact_rolling(res, cp.pivotB, posB, ornB, mk3(d.angvel[b]), d.dt);
        if (nearest < res.num && !(merged >> nearest & 1u)) { merge_point(res.pt[nearest], cp, ornA, ornB); merged |= 1u << nearest; }
        else {                                          // should_remove_point, collision_util.cpp:397-413
            v3 pA = to_world(cp.pivotA, posA, ornA), pB = to_world(cp.pivotB, posB, ornB);
            v3 dd = pA - pB;
            float nd = dot(dd, cp.normal);
            v3 td = dd - nd * cp.normal;
            if (nd > BREAKING_THRESHOLD || length_sqr(td) > BREAKING_THRESHOLD * BREAKING_THRESHOLD) continue;
            cp.distance = dot(cp.normal, pA - pB);      // update_contact_distances
        }
        keep |= 1u << s;
        store_point(d, m, s, cp);
    }
    int num = __popc(keep);
    if (keep != (1u << num0) - 1u || merged != (1u << res.num) - 1u) num = np_rearrange(d, m, pr, res, keep, merged);
    d.mstate[m] = (st & ~MS_NPTS_MASK) | (uint32_t)num;
    // the island rebuild reads whether a manifold has points (colouring, island census) and, on the dataflow path,
    // its point count (sort key); inside an island tile the count only matters to the solver itself, except that a
    // two-point tile has no room for a third point
    const uint32_t was = st & MS_NPTS_MASK;
    if ((uint32_t)num != was) {
        const uint32_t tile = d.btile[key_body(d, pr)];
        if (was == 0u || num == 0 || tile == TILE_NONE || (num > 2 && was <= 2u && tile < d.cnt->ntiles2)) d.cnt->graph_changed = 1u;
    }
}
// detect_collision (collision_util.cpp:440-475) of the manifold at position i of the sorted list, then its np_merge.
// FN is the ordered pair type of the launch, 0 in the light launch, which takes it from the shapes at run time.  Sleeping
// manifolds are not in the list: their points and lifetimes stay untouched.
template <int FN>
B2D_D void np_run(int fn, float4 A, float4 B, const CCtx &c, CResult &r) {
    if constexpr (FN != 0) run_pair(FN, A, B, c, r); else run_light_pair(fn, A, B, c, r);
}
template <int FN>
B2D_D void np_manifold(const Dev &d, uint32_t i) {
    const uint32_t m = d.npidx[i];
    const uint32_t st = d.mstate[m];
    const uint2 pr = d.mpair[m];
    const uint32_t fa = d.flags[pr.x], fb = d.flags[pr.y];
    // the AABB gate, collision_util.cpp:444-474; a manifold it closes still merges an empty result into its points
    const bool near = intersect(inset(body_box(d, pr.x), -BREAKING_THRESHOLD), body_box(d, pr.y));
    if (!near && !(st & MS_NPTS_MASK)) return;
    const v3 posA = mk3(d.pos[pr.x]), posB = mk3(d.pos[pr.y]);
    const q4 ornA = mkq(d.orn[pr.x]), ornB = mkq(d.orn[pr.y]);
    CResult res; res.num = 0;
    if (near) {
        const int ka = shape_of(fa), kb = shape_of(fb);
        const int fn = pair_fn(ka, kb);             // the list holds type FN = pair_fn(ka, kb), or pair_fn(kb, ka) if that is 0
        CCtx ctx; ctx.threshold = COLLISION_THRESHOLD;
        if (fn) {
            ctx.posA = posA; ctx.ornA = ornA; ctx.posB = posB; ctx.ornB = ornB;
            np_run<FN>(fn, d.shp[pr.x], d.shp[pr.y], ctx, res);
        } else {                                    // swap_collide, collide.hpp:369-374
            ctx.posA = posB; ctx.ornA = ornB; ctx.posB = posA; ctx.ornB = ornA;
            np_run<FN>(pair_fn(kb, ka), d.shp[pr.y], d.shp[pr.x], ctx, res);
            swap_result(res);
        }
    }
    np_merge(d, m, res);
}
// the two heavy overloads (box-box, capsule-box) get a launch each over their range of the list.  The launch bounds
// hold the residency the collide code needs (3, 4 and, for the light kernel, 6 CTAs per SM), so that the merge's
// cold insertion path does not raise the register count for everyone
template <int FN>
__global__ void __launch_bounds__(128, FN == 5 ? 3 : 4) k_np_collide(Dev d) {
    const uint32_t b = d.cnt->npoff[FN], e = d.cnt->npoff[FN + 1];
    for (uint32_t i = b + blockIdx.x * blockDim.x + threadIdx.x; i < e; i += gridDim.x * blockDim.x) np_manifold<FN>(d, i);
}
// the seven light ones share one: types 1-4 and 6-8, two ranges of the list walked as one
__global__ void __launch_bounds__(128, 6) k_np_collide_light(Dev d) {
    const uint32_t b0 = d.cnt->npoff[1], n0 = d.cnt->npoff[5] - b0, b1 = d.cnt->npoff[6], n = n0 + d.cnt->npoff[9] - b1;
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) np_manifold<0>(d, j < n0 ? b0 + j : b1 + (j - n0));
}

// ====================================================================== islands (connected components)

// Union-find with atomic hooking (roots hook onto smaller ids, so every component ends labelled by its
// smallest body id).  Only procedural nodes connect (core/entity_graph.hpp:303-307); every manifold is an
// edge even with zero points (make_contact_manifold adds a null_constraint edge), plus every joint.
B2D_D uint32_t cc_find(uint32_t *parent, uint32_t x) {
    uint32_t p = parent[x];
    while (p != x) { uint32_t gp = parent[p]; if (gp != p) parent[x] = gp; x = p; p = parent[x]; }
    return x;
}
B2D_D void cc_union(uint32_t *parent, uint32_t a, uint32_t b) {
    for (;;) {
        a = cc_find(parent, a); b = cc_find(parent, b);
        if (a == b) return;
        if (a < b) { uint32_t t = a; a = b; b = t; }
        uint32_t old = atomicCAS(&parent[a], a, b);
        if (old == a) return;
    }
}
__global__ void k_cc_init(Dev d) { GRID_STRIDE(i, d.nbodies) d.parent[i] = i; }
// one atomic per distinct address per warp (a pile is ONE island: 262 144 lanes would otherwise queue on one word)
B2D_D void island_count(uint32_t *ctr, uint32_t root) {
    const uint32_t grp = __match_any_sync(__activemask(), root);
    if ((threadIdx.x & 31u) == (uint32_t)(__ffs(grp) - 1)) atomicAdd(&ctr[root], (uint32_t)__popc(grp));
}
// Two rounds: a quarter of the edges is hooked first and the forest flattened; in a dense contact graph that already
// joins most of every island, so the remaining edges mostly find parent[a] == parent[b] with two plain reads and never
// reach the find / compare-and-swap path (which otherwise funnels the whole grid through the root of a giant island).
__global__ void k_cc_union(Dev d, int round) {
    const uint32_t hwm = d.cnt->hwm;
    GRID_STRIDE(m, hwm + d.nhinges) {
        uint2 p;
        if (m < hwm) {
            if (((m & 3u) == 0u) != (round == 0)) continue;
            if (!(d.mstate[m] & MS_ALIVE)) continue;
            p = d.mpair[m];
        } else { if (round != 0) continue; p = d.hpair[m - hwm]; }
        if (!is_procedural(d.flags[p.x]) || !is_procedural(d.flags[p.y])) continue;
        if (round != 0 && d.parent[p.x] == d.parent[p.y]) continue;
        cc_union(d.parent, p.x, p.y);
    }
}
__global__ void k_cc_flatten(Dev d, int last) {
    GRID_STRIDE(i, d.nbodies) {
        if (is_procedural(d.flags[i])) {
            // read-only walk: a concurrent path-compressing find could overwrite another thread's final root with a
            // stale grandparent; writing the root itself is harmless to walkers passing through i
            uint32_t r = i, p = d.parent[r];
            while (p != r) { r = p; p = d.parent[r]; }
            d.parent[i] = r;
            if (last && r == i) atomicAdd(&d.cnt->nislands, 1u);
        }
        else if (last) d.parent[i] = 0xFFFFFFFFu;
    }
}

// ---- island sleeping: wake_up_islands + put_islands_to_sleep (island_manager.cpp:524-539, :568-623) on labels that are
// recomputed every step.  island::sleep_timestamp follows the island the way merge_islands (:303-316, biggest
// constituent survives) and split_islands (:431-447, biggest part keeps the entity) move it: a new island takes the
// timestamp of its biggest previous constituent O (procedural-body count, ties to the smaller label) iff it is also
// O's biggest heir.  An island with an awake and a sleeping member was just joined by a new edge: everybody wakes
// (insert_to_island -> wake_up_island, :257-295).  isl_flags: 1 any awake, 2 any fast, 4 falls asleep now.
constexpr float PI_F = 3.1415926535897932384626433832795029f;   // math/constants.hpp
constexpr float SLEEP_LIN2 = 0.005f * 0.005f;                      // config/constants.hpp:41-42
constexpr float SLEEP_ANG2 = (PI_F / 48.0f) * (PI_F / 48.0f);
__global__ void k_sleep_gather(Dev d) {
    GRID_STRIDE(i, d.nbodies) {
        const uint32_t f = d.flags[i];
        if (!is_procedural(f)) continue;
        const uint32_t r = d.parent[i];
        atomicAdd(&d.size_new[r], 1u);
        uint32_t bits = (f & F_SLEEPING) ? 0u : 1u;
        const v3 v = mk3(d.linvel[i]), w = mk3(d.angvel[i]);
        if (length_sqr(v) > SLEEP_LIN2 || length_sqr(w) > SLEEP_ANG2) bits |= 2u;
        if (bits) atomicOr(&d.isl_flags[r], bits);
        const uint32_t o = d.prev_label[i];
        if (o != 0xFFFFFFFFu) atomicMax(&d.contributor[r], ((unsigned long long)d.isl_size[o] << 32) | (unsigned long long)(~o));
    }
}
__global__ void k_sleep_heirs(Dev d) {
    GRID_STRIDE(i, d.nbodies) {
        if (!is_procedural(d.flags[i])) continue;
        const uint32_t o = d.prev_label[i], r = d.parent[i];
        if (o != 0xFFFFFFFFu) atomicMax(&d.heir[o], ((unsigned long long)d.size_new[r] << 32) | (unsigned long long)(~r));
    }
}
__global__ void k_sleep_decide(Dev d, double last_time) {
    GRID_STRIDE(r, d.nbodies) {
        double ts = -1.0;
        const uint32_t fl = d.isl_flags[r];
        if (d.size_new[r] && (fl & 1u)) {                      // sleeping islands are not visited (exclude_sleeping_disabled)
            const unsigned long long c = d.contributor[r];
            if (c) {
                const uint32_t o = ~(uint32_t)(c & 0xFFFFFFFFull);
                if (~(uint32_t)(d.heir[o] & 0xFFFFFFFFull) == r) ts = d.isl_ts[o];
            }
            if (!(fl & 2u)) {
                if (ts < 0) ts = last_time;
                else if (last_time - ts > 2.0) { d.isl_flags[r] = fl | 4u; ts = -1.0; }      // island_time_to_sleep
            } else ts = -1.0;
        }
        d.ts_new[r] = ts;
    }
}
__global__ void k_sleep_apply(Dev d) {
    GRID_STRIDE(i, d.nbodies) {
        uint32_t f = d.flags[i];
        if (!is_procedural(f)) { d.prev_label[i] = 0xFFFFFFFFu; continue; }
        const uint32_t r = d.parent[i], fl = d.isl_flags[r];
        if (fl & 1u) f &= ~F_SLEEPING;
        if (fl & 4u) { f |= F_SLEEPING; d.linvel[i] = make_float4(0, 0, 0, 0); d.angvel[i] = make_float4(0, 0, 0, 0); }     // put_to_sleep, :541-566
        if (f != d.flags[i]) d.cnt->graph_changed = 1u;          // a body fell asleep or woke up
        d.flags[i] = f;
        d.prev_label[i] = r;
    }
}
// wake_up_entity (util/island_util.cpp): the island follows at the next island update
__global__ void k_wake_bodies(Dev d, const uint32_t *ids, uint32_t n) {
    GRID_STRIDE(k, n) { const uint32_t i = ids ? ids[k] : k; d.flags[i] &= ~F_SLEEPING; }
}

// ====================================================================== solver: gravity, colouring

// apply_gravity, sys/apply_gravity.hpp:12-17
__global__ void k_gravity(Dev d) {
    GRID_STRIDE(i, d.nbodies) {
        if (!is_dynamic(d.flags[i])) continue;
        v3 v = mk3(d.linvel[i]); v += mk3(d.grav[i]) * d.dt;
        d.linvel[i] = f4(v, 0);
    }
}
// First kernel of the island rebuild after the connected components: resets what the colouring and the tile packing
// accumulate into (they run after this kernel), counts the dynamic bodies per island and clears the rebuild flag.
__global__ void k_island_census(Dev d) {
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        Counters &c = *d.cnt;
        c.remaining[0] = c.remaining[1] = 0; c.nlist = 0; c.bar = 0; c.tile_wmax = 0; c.ncolors_all = 0; c.nhcolors_all = 0;
        c.graph_changed = 0u;
    }
    GRID_STRIDE(i, d.nbodies) {
        d.bmask[i] = 0ULL; d.jmask[i] = 0ULL; d.prop[i] = ~0ULL; d.jprop[i] = ~0ULL;
        if (!is_dynamic(d.flags[i])) continue;
        island_count(d.isl_nb, d.parent[i]);          // census for the island tiles (zeroed by the host, k_tile_weights)
    }
}
#ifndef B2D_EMU
// Head of the conditional graph node around the island rebuild: run it iff something it reads changed.
__global__ void k_rebuild_decide(Dev d, cudaGraphConditionalHandle h) {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    Counters &c = *d.cnt;
    const bool changed = c.graph_changed != 0u;
    cudaGraphSetConditional(h, changed ? 1u : 0u);
    if (changed) ++c.steps_rebuilt; else ++c.steps_reused;
}
#endif

// Colours persist from step to step for constraints that keep producing rows, so in steady state only the few
// manifolds that just gained their first point (and new hinges) enter the colouring rounds.  This pass
// releases the colour of manifolds that lost all points, rebuilds the per-body "colours in use" masks from
// the constraints that keep theirs (masks are zeroed by the host before the launch) and lists the uncoloured
// ones.  With recolor != 0 everything is recoloured from scratch.
__global__ void k_color_list(Dev d, int recolor) {
    const uint32_t hwm = d.cnt->hwm;
    GRID_STRIDE(m, hwm) {
        uint32_t st = d.mstate[m];
        if (!(st & MS_ALIVE)) continue;
        uint32_t col = (st >> MS_COLOR_SHIFT) & 0xFFu;
        if (!(st & MS_NPTS_MASK) || recolor) {
            if (col != COLOR_NONE) { st |= MS_COLOR_MASK; d.mstate[m] = st; col = COLOR_NONE; }
            if (!(st & MS_NPTS_MASK)) continue;
        }
        const uint2 p = d.mpair[m];
        const bool da = is_dynamic(d.flags[p.x]), db = is_dynamic(d.flags[p.y]);
        if (!da && !db) {          // sleeping: drops its colour, takes a fresh one when the island wakes
            if (col != COLOR_NONE) d.mstate[m] = st | MS_COLOR_MASK;
            continue;
        }
        if (col == COLOR_NONE) { uint32_t k = atomicAdd(&d.cnt->nlist, 1u); d.clist[k] = m; }
        else {
            if (da) atomicOr(&d.bmask[p.x], 1ULL << col);
            if (db) atomicOr(&d.bmask[p.y], 1ULL << col);
        }
        const uint32_t root = d.parent[da ? p.x : p.y];
        island_count(d.isl_nm, root);
        {   // one atomic per island per warp, as in island_count (a pile of boxes is one island)
            const uint32_t grp = __match_any_sync(__activemask(), root), multi = __ballot_sync(__activemask(), (st & MS_NPTS_MASK) > 2u);
            if ((grp & multi) && (threadIdx.x & 31u) == (uint32_t)(__ffs(grp) - 1)) atomicOr(&d.isl_nm[root], ISL_MULTIPOINT);
        }
    }
    GRID_STRIDE(h, d.nhinges) {
        uint2 p = d.hpair[h];
        const bool da = is_dynamic(d.flags[p.x]), db = is_dynamic(d.flags[p.y]);
        if (recolor || (!da && !db)) d.hcolor[h] = COLOR_NONE;
        if (da || db) island_count(d.isl_nh, d.parent[da ? p.x : p.y]);
        uint32_t col = d.hcolor[h];
        if (col == COLOR_NONE) continue;
        if (da) atomicOr(&d.jmask[p.x], 1ULL << col);
        if (db) atomicOr(&d.jmask[p.y], 1ULL << col);
    }
}

// Deterministic greedy colouring of the constraint graph (manifolds and hinges are coloured independently:
// they are solved in separate passes).  Jones-Plassmann style rounds over the uncoloured constraints: one
// takes the lowest colour unused on either of its dynamic bodies once it holds the smallest (hashed) priority
// among the still uncoloured constraints on both bodies.  Priorities depend only on the slot index and the
// inputs are the previous (deterministic) colouring, so the Gauss-Seidel order is reproducible run to run.
__global__ void __launch_bounds__(256) k_color(Dev d) {
    GridBarrier grid(&d.cnt->bar);
    Counters &c = *d.cnt;
    const uint32_t nlist = c.nlist;
    const uint32_t total = nlist + d.nhinges;
    for (uint32_t round = 0;; ++round) {
        const unsigned long long stamp = (unsigned long long)(0xFFFFu - (round & 0xFFFFu)) << 48;
        GRID_STRIDE(k, total) {
            const bool isM = k < nlist;
            uint32_t id; uint2 p; unsigned long long *prop;
            if (isM) { id = d.clist[k]; if (((d.mstate[id] >> MS_COLOR_SHIFT) & 0xFFu) != COLOR_NONE) continue; p = d.mpair[id]; prop = d.prop; }
            else { id = k - nlist; if (d.hcolor[id] != COLOR_NONE) continue; p = d.hpair[id]; prop = d.jprop; if (!is_dynamic(d.flags[p.x]) && !is_dynamic(d.flags[p.y])) continue; }
            unsigned long long v = stamp | ((unsigned long long)(hash64(id) & 0x3FFFFFu) << 26) | id;
            if (is_dynamic(d.flags[p.x])) atomicMin(&prop[p.x], v);
            if (is_dynamic(d.flags[p.y])) atomicMin(&prop[p.y], v);
        }
        grid.sync();
        GRID_STRIDE(k, total) {
            const bool isM = k < nlist;
            uint32_t id; uint2 p; unsigned long long *prop, *mask;
            if (isM) { id = d.clist[k]; if (((d.mstate[id] >> MS_COLOR_SHIFT) & 0xFFu) != COLOR_NONE) continue; p = d.mpair[id]; prop = d.prop; mask = d.bmask; }
            else { id = k - nlist; if (d.hcolor[id] != COLOR_NONE) continue; p = d.hpair[id]; prop = d.jprop; mask = d.jmask; if (!is_dynamic(d.flags[p.x]) && !is_dynamic(d.flags[p.y])) continue; }
            unsigned long long v = stamp | ((unsigned long long)(hash64(id) & 0x3FFFFFu) << 26) | id;
            bool da = is_dynamic(d.flags[p.x]), db = is_dynamic(d.flags[p.y]);
            bool win = (!da || prop[p.x] == v) && (!db || prop[p.y] == v);
            if (win) {
                unsigned long long used = (da ? mask[p.x] : 0ULL) | (db ? mask[p.y] : 0ULL);
                unsigned long long freeb = ~used;
                uint32_t col = freeb ? (uint32_t)(__ffsll((long long)freeb) - 1) : (MAX_COLORS - 1);
                if (!freeb) atomicOr(&c.err, ERR_COLOR_OVERFLOW);
                if (da) atomicOr(&mask[p.x], 1ULL << col);
                if (db) atomicOr(&mask[p.y], 1ULL << col);
                if (isM) d.mstate[id] = (d.mstate[id] & ~MS_COLOR_MASK) | (col << MS_COLOR_SHIFT);
                else d.hcolor[id] = col;
            } else atomicAdd(&c.remaining[round & 1], 1u);
        }
        grid.sync();
        uint32_t rem = c.remaining[round & 1];
        if (blockIdx.x == 0 && threadIdx.x == 0) c.remaining[(round + 1) & 1] = 0;
        if (rem == 0) break;
        grid.sync();
    }
}

// ---- island tiles.  An island with at most TILE_ISLAND_MAX dynamic bodies, manifolds with points and joints is solved
// inside one CTA (k_island_tiles).  Islands are packed into tiles in root-id order: with weight
// w = max(bodies, manifolds, joints) <= TILE_ISLAND_MAX per island and P the exclusive prefix sum of the weights, island
// -> tile P / g with g = TILE_CAP + 1 - (heaviest tiled island) puts at most TILE_CAP of each into every tile.  Which islands
// are tiled changes speed, never results: the per-body constraint order is fixed by the colours alone.
// Two classes, each packed this way in root order: two-point islands (no manifold with more than 2 points: spheres,
// capsules, planes) in tiles [0, ntiles2), solved by the two-point kernel, then the others in [ntiles2, ntiles).  The
// two prefix sums are the two words of one 64-bit scan.
__global__ void k_tile_weights(Dev d) {
    uint32_t wmax = 0;
    GRID_STRIDE(i, d.nbodies) {
        uint32_t w = 0;
        bool multi = false;
        if (is_dynamic(d.flags[i]) && d.parent[i] == i) {
            const uint32_t nb = d.isl_nb[i], nm = d.isl_nm[i] & ~ISL_MULTIPOINT, nh = d.isl_nh[i];
            multi = (d.isl_nm[i] & ISL_MULTIPOINT) != 0u;
            if (nb <= TILE_ISLAND_MAX && nm <= TILE_ISLAND_MAX && nh <= TILE_ISLAND_MAX && (nm | nh)) w = max(nb, max(nm, nh));
        }
        d.swgt[i] = multi ? (unsigned long long)w << 32 : w;
        wmax = max(wmax, w);
    }
    wmax = __reduce_max_sync(0xffffffffu, wmax);
    if ((threadIdx.x & 31u) == 0 && wmax) atomicMax(&d.cnt->tile_wmax, wmax);
}
// islands start a new tile every `granule` units of weight: a tile then holds less than granule + heaviest island <= TILE_CAP
B2D_D uint32_t tile_granule(const Dev &d) { return (uint32_t)TILE_CAP + 1u - max(d.cnt->tile_wmax, 1u); }
__global__ void k_tile_assign(Dev d) {
    const uint32_t n = d.nbodies, g = tile_granule(d);
    const unsigned long long total = d.swsum[n - 1] + d.swgt[n - 1];
    const uint32_t ntiles2 = ((uint32_t)total + g - 1) / g;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        d.cnt->ntiles2 = min(d.max_tiles, ntiles2);
        d.cnt->ntiles = min(d.max_tiles, ntiles2 + ((uint32_t)(total >> 32) + g - 1) / g);
    }
    GRID_STRIDE(i, n) {
        uint32_t tile = TILE_NONE, slot = SLOT_NONE;
        if (is_dynamic(d.flags[i])) {
            const uint32_t r = d.parent[i];
            if (d.swgt[r]) {
                const unsigned long long p = d.swsum[r];
                tile = (d.swgt[r] >> 32) ? ntiles2 + (uint32_t)(p >> 32) / g : (uint32_t)p / g;
                if (tile < d.max_tiles) {                           // order within the tile is immaterial; one atomic per tile per warp
                    const uint32_t grp = __match_any_sync(__activemask(), tile), lane = threadIdx.x & 31u, leader = (uint32_t)(__ffs(grp) - 1);
                    uint32_t base = 0;
                    if (lane == leader) base = atomicAdd(&d.tile_nb[tile], (uint32_t)__popc(grp));
                    slot = __shfl_sync(grp, base, leader) + __popc(grp & ((1u << lane) - 1u));
                    d.tile_body[(size_t)tile * TILE_CAP + slot] = i;
                } else tile = TILE_NONE;
            }
        }
        d.btile[i] = tile; d.bslot[i] = slot;
    }
}
// Sort keys.  Tiled constraints first, tile-major then colour; then the dataflow path's constraints by colour, point
// count (a chunk of 32 manifolds runs the same number of row solves in every lane) and the spatial rank of the
// manifold's dynamic body (lanes of a chunk touch neighbouring bodies, whose predecessors finish at about the same
// time and whose records share L2 sectors); constraints without rows this step last.
__global__ void k_color_keys(Dev d) {
    const uint32_t hwm = d.cnt->hwm;
    uint32_t cmax = 0, hmax = 0;
    GRID_STRIDE(m, d.NM) {
        uint32_t key = KEY_INACTIVE;
        if (m < hwm) {
            uint32_t st = d.mstate[m];
            if ((st & MS_ALIVE) && (st & MS_NPTS_MASK) && ((st >> MS_COLOR_SHIFT) & 0xFFu) != COLOR_NONE) {      // uncoloured = sleeping
                const uint2 pr = d.mpair[m];
                const uint32_t b = key_body(d, pr), col = (st >> MS_COLOR_SHIFT) & 0x3Fu;
                const uint32_t tile = d.btile[b];
                cmax = max(cmax, col + 1u);
                if (tile != TILE_NONE) key = (tile << 6) | col;
                else {
                    key = KEY_DF | (col << KEY_DF_COLOR_SHIFT) | (((st & MS_NPTS_MASK) - 1u) << KEY_DF_SPATIAL_BITS) | df_spatial(d, d.brank[b]);
                }
            }
        }
        d.ckey[m] = key; d.cidx[m] = m;
    }
    GRID_STRIDE(h, d.NH) {
        uint32_t key = KEY_INACTIVE;
        if (h < d.nhinges) {
            const uint2 p = d.hpair[h];
            if (is_dynamic(d.flags[p.x]) || is_dynamic(d.flags[p.y])) {
                const uint32_t tile = d.btile[is_dynamic(d.flags[p.x]) ? p.x : p.y], col = d.hcolor[h] & 0x3Fu;
                hmax = max(hmax, col + 1u);
                key = tile != TILE_NONE ? ((tile << 6) | col) : (KEY_DF | (col << KEY_DF_COLOR_SHIFT));
            }
        }
        d.hkey[h] = key; d.hidx[h] = h;
    }
    cmax = __reduce_max_sync(0xffffffffu, cmax); hmax = __reduce_max_sync(0xffffffffu, hmax);
    if ((threadIdx.x & 31u) == 0) { if (cmax) atomicMax(&d.cnt->ncolors_all, cmax); if (hmax) atomicMax(&d.cnt->nhcolors_all, hmax); }
    if (blockIdx.x == 0 && threadIdx.x < MAX_COLORS + 2) { d.cnt->coff[threadIdx.x] = 0xFFFFFFFFu; d.cnt->hoff[threadIdx.x] = 0xFFFFFFFFu; }
    if (blockIdx.x == 0 && threadIdx.x == 0) { Counters &c = *d.cnt; c.nactive = d.NM; c.nhactive = d.NH; c.ntiled = 0xFFFFFFFFu; c.nhtiled = 0xFFFFFFFFu; }
}
// Range boundaries in the sorted arrays: [tile_c0, tile_c1) per tile (preset to empty by the host), the start of each
// dataflow colour, the first constraint without rows.
B2D_D void key_boundary(uint32_t i, uint32_t prev, uint32_t key, bool first, uint32_t *t0, uint32_t *t1, uint32_t *off, uint32_t *ntiled, uint32_t *nact) {
    const uint32_t cls = key >> (KEY_TILE_BITS + 6), pcls = prev >> (KEY_TILE_BITS + 6);      // 0 tiled, 1 dataflow, 2 inactive
    if (cls == 0) {
        if (first || (prev >> 6) != (key >> 6)) { t0[key >> 6] = i; if (!first) t1[prev >> 6] = i; }
        return;
    }
    if (!first && pcls == 0) t1[prev >> 6] = i;                                                   // the last tile ends here
    if (first || pcls != cls) { if (cls == 1) *ntiled = i; else { *nact = i; if (first || pcls == 0) *ntiled = i; } }
    if (cls == 1) { const uint32_t col = (key >> KEY_DF_COLOR_SHIFT) & 63u; if (first || pcls != 1 || ((prev >> KEY_DF_COLOR_SHIFT) & 63u) != col) off[col] = i; }
}
__global__ void k_color_offsets(Dev d) {
    Counters &c = *d.cnt;
    GRID_STRIDE(i, d.NM) key_boundary(i, i ? d.ckey_s[i - 1] : 0u, d.ckey_s[i], i == 0, d.tile_c0, d.tile_c1, c.coff, &c.ntiled, &c.nactive);
    GRID_STRIDE(i, d.NH) key_boundary(i, i ? d.hkey_s[i - 1] : 0u, d.hkey_s[i], i == 0, d.tile_h0, d.tile_h1, c.hoff, &c.nhtiled, &c.nhactive);
}
__global__ void k_color_fixup(Dev d) {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    Counters &c = *d.cnt;
    // every entry has rows: no boundary was seen (presets: nactive = capacity, ntiled = 0xFFFFFFFF)
    if (c.ntiled == 0xFFFFFFFFu) c.ntiled = c.nactive;
    if (c.nhtiled == 0xFFFFFFFFu) c.nhtiled = c.nhactive;
    // the last tile runs to the end of the tiled range when nothing follows it (no boundary closes it)
    if (c.ntiles) {
        if (c.ntiled && d.ckey_s[c.ntiled - 1] >> (KEY_TILE_BITS + 6) == 0) d.tile_c1[d.ckey_s[c.ntiled - 1] >> 6] = c.ntiled;
        if (c.nhtiled && d.hkey_s[c.nhtiled - 1] >> (KEY_TILE_BITS + 6) == 0) d.tile_h1[d.hkey_s[c.nhtiled - 1] >> 6] = c.nhtiled;
    }
    c.coff[MAX_COLORS] = c.nactive; c.hoff[MAX_COLORS] = c.nhactive;
    c.coff[MAX_COLORS + 1] = c.coff[MAX_COLORS]; c.hoff[MAX_COLORS + 1] = c.hoff[MAX_COLORS];
    uint32_t nc = 0, nh = 0;
    for (int k = MAX_COLORS - 1; k >= 0; --k) {
        if (c.coff[k] == 0xFFFFFFFFu) c.coff[k] = c.coff[k + 1]; else if (!nc) nc = k + 1;
        if (c.hoff[k] == 0xFFFFFFFFu) c.hoff[k] = c.hoff[k + 1]; else if (!nh) nh = k + 1;
    }
    c.ncolors = nc; c.nhcolors = nh;
    c.cchunk[0] = 0; c.hchunk[0] = 0;
    for (int k = 0; k <= MAX_COLORS; ++k) {
        c.cchunk[k + 1] = c.cchunk[k] + (k < (int)nc ? (c.coff[k + 1] - c.coff[k] + 31) / 32 : 0);
        c.hchunk[k + 1] = c.hchunk[k] + (k < (int)nh ? (c.hoff[k + 1] - c.hoff[k] + 31) / 32 : 0);
    }
}

// ====================================================================== solver: row preparation

struct SBody { v3 v, w; float inv_m; m3 inv_I; bool proc; };
// constraint_body + row masses, solver.cpp:101-147: dynamic -> (inv_m, inv_IW, v, w); kinematic -> (0, 0, v, w);
// static -> zeros.
B2D_D SBody solver_body(const Dev &d, uint32_t i, uint32_t f) {
    SBody s;
    s.proc = is_dynamic(f);
    if (s.proc) { float4 r0 = d.invIW[3 * i]; s.inv_m = r0.w; s.inv_I.r0 = mk3(r0); s.inv_I.r1 = mk3(d.invIW[3 * i + 1]); s.inv_I.r2 = mk3(d.invIW[3 * i + 2]); }
    else { s.inv_m = 0; s.inv_I = m3_zero(); }
    if (kind_of(f) == 2u) { s.v = mk3(0, 0, 0); s.w = mk3(0, 0, 0); } else { s.v = mk3(d.linvel[i]); s.w = mk3(d.angvel[i]); }
    return s;
}
// get_effective_mass / prepare_row, util/constraint_util.cpp:137-146, constraints/constraint_row.cpp:6-22
B2D_D float eff_mass(v3 J0, v3 J1, v3 J2, v3 J3, const SBody &A, const SBody &B) {
    float s = dot(J0, J0) * A.inv_m + dot(A.inv_I * J1, J1) + dot(J2, J2) * B.inv_m + dot(B.inv_I * J3, J3);
    return 1.0f / s;
}
B2D_D float rel_speed(v3 J0, v3 J1, v3 J2, v3 J3, v3 vA, v3 wA, v3 vB, v3 wB) {
    return dot(J0, vA) + dot(J1, wA) + dot(J2, vB) + dot(J3, wB);
}

// contact_constraint::prepare (contact_constraint.cpp:15-56) + prepare_row of contact point slot mi: r0 = normal | rhs,
// r1 = rA | eff_mass, r2 = rB | friction, r3 = eff_mass t0, t1, rhs t0, t1, im = warm-start impulses (n, t0, t1).
// Row storage keeps (n, rA, rB) and rebuilds the Jacobian in registers: 84 B/point instead of the reference's 312 B
// (constraint_row + _friction).  Shared by k_prepare_contacts, k_island_tiles and the restitution solver, so all produce
// the same bits.  `restitution`: the rows of the restitution solver's groups (constraint_row_options{}, restitution_solver.cpp:
// 146-310): no penetration error, the point's restitution always applied, no warm start.
B2D_D void contact_point_rows(const Dev &d, size_t mi, const SBody &A, const SBody &B, v3 posA, q4 ornA, v3 posB, q4 ornB,
                              float4 &r0, float4 &r1, float4 &r2, float4 &r3, float4 &imp, bool restitution = false) {
    float4 a4 = d.pA[mi], b4 = d.pB[mi], n4 = d.pN[mi], im = restitution ? make_float4(0, 0, 0, 0) : d.pI[mi];
    v3 normal = mk3(n4);
    v3 pAw = to_world(mk3(a4), posA, ornA), pBw = to_world(mk3(b4), posB, ornB);
    v3 rA = pAw - posA, rB = pBw - posB;
    v3 J1 = cross(rA, normal), J2 = -normal, J3 = -cross(rB, normal);
    float em = eff_mass(normal, J1, J2, J3, A, B);
    float error = 0.0f;
    if (!restitution && a4.w > 0) error = a4.w / d.dt;
    float relvel = rel_speed(normal, J1, J2, J3, A.v, A.w, B.v, B.w);
    // solver.cpp:217-236: with the restitution solver on, the ordinary rows carry no restitution
    float rhs = -(error * 0.2f + relvel * (1.0f + (restitution ? n4.w : (d.rest_iters ? 0.0f : n4.w))));
    v3 t, u; plane_space(normal, t, u);
    v3 T1 = cross(rA, t), T2 = -t, T3 = -cross(rB, t);
    v3 U1 = cross(rA, u), U2 = -u, U3 = -cross(rB, u);
    float em_t = eff_mass(t, T1, T2, T3, A, B), em_u = eff_mass(u, U1, U2, U3, A, B);
    float rhs_t = -rel_speed(t, T1, T2, T3, A.v, A.w, B.v, B.w), rhs_u = -rel_speed(u, U1, U2, U3, A.v, A.w, B.v, B.w);
    r0 = f4(normal, rhs); r1 = f4(rA, em); r2 = f4(rB, b4.w);
    r3 = make_float4(em_t, em_u, rhs_t, rhs_u);
    imp = make_float4(im.x, im.y, im.z, 0);
}

// hinge_constraint::prepare, hinge_constraint.cpp:26-69 (no limits / springs / torque rows): the 7 row vectors of hinge h
// (rA | em0, rB | em1, p | em2, q | em3, em4 rhs0 rhs1 rhs2, rhs3 rhs4 imp0 imp1, imp2 imp3 imp4) to R[0], R[stride], ...
// Shared by k_prepare_hinges and k_island_tiles.
B2D_D void hinge_rows(const Dev &d, uint32_t h, const SBody &A, const SBody &B, v3 posA, q4 ornA, v3 posB, q4 ornB,
                      float4 *R, uint32_t stride) {
    v3 rA = to_world(mk3(d.hpivA[h]), posA, ornA) - posA;
    v3 rB = to_world(mk3(d.hpivB[h]), posB, ornB) - posB;
    v3 p = rotate(ornA, mk3(d.hfA1[h])), q = rotate(ornA, mk3(d.hfA2[h]));
    float em[5], rhs[5];
    #pragma unroll
    for (int k = 0; k < 3; ++k) {
        v3 e = axis_vec(k);
        // rows of skew(r): (0,-z,y), (z,0,-x), (-y,x,0)  matrix3x3.hpp:243-249
        v3 sa = k == 0 ? mk3(0, -rA.z, rA.y) : (k == 1 ? mk3(rA.z, 0, -rA.x) : mk3(-rA.y, rA.x, 0));
        v3 sb = k == 0 ? mk3(0, -rB.z, rB.y) : (k == 1 ? mk3(rB.z, 0, -rB.x) : mk3(-rB.y, rB.x, 0));
        v3 J1 = -sa, J2 = -e, J3 = sb;
        em[k] = eff_mass(e, J1, J2, J3, A, B);
        rhs[k] = -(0.0f * 0.2f + rel_speed(e, J1, J2, J3, A.v, A.w, B.v, B.w) * (1.0f + 0.0f));
    }
    const v3 z = mk3(0, 0, 0);
    em[3] = eff_mass(z, p, z, -p, A, B); rhs[3] = -(0.0f * 0.2f + rel_speed(z, p, z, -p, A.v, A.w, B.v, B.w) * (1.0f + 0.0f));
    em[4] = eff_mass(z, q, z, -q, A, B); rhs[4] = -(0.0f * 0.2f + rel_speed(z, q, z, -q, A.v, A.w, B.v, B.w) * (1.0f + 0.0f));
    const float *imp = d.himp + 5 * (size_t)h;
    R[0] = f4(rA, em[0]); R[stride] = f4(rB, em[1]); R[2 * stride] = f4(p, em[2]); R[3 * stride] = f4(q, em[3]);
    R[4 * stride] = make_float4(em[4], rhs[0], rhs[1], rhs[2]);
    R[5 * stride] = make_float4(rhs[3], rhs[4], imp[0], imp[1]);
    R[6 * stride] = make_float4(imp[2], imp[3], imp[4], 0);
}

// Row header of a sorted constraint (Dev::hdr / hhdr): the tags of bodies a and b, the point count or hinge id, and the
// bodies' slots in an island tile.  A body tag is the body id, with the top bit set for a body the solver does not move.
B2D_D uint32_t body_tag(uint32_t id, const SBody &b) { return id | (b.proc ? 0u : 0x80000000u); }
B2D_D uint32_t tag_id(uint32_t tag) { return tag & 0x7FFFFFFFu; }
B2D_D bool tag_proc(uint32_t tag) { return !(tag >> 31); }
B2D_D uint32_t slot_pair(uint32_t sa, uint32_t sb) { return sa | (sb << 16); }
B2D_D uint32_t slot_a(uint32_t pair) { return pair & 0xFFFFu; }
B2D_D uint32_t slot_b(uint32_t pair) { return pair >> 16; }
// island label of a constraint between bodies a and b (the dynamic one's)
B2D_D uint32_t island_of(const Dev &d, uint32_t a, uint32_t b) { uint32_t l = d.parent[a]; return l != 0xFFFFFFFFu ? l : d.parent[b]; }

// Dataflow tickets (k_solve_df, k_position_df): per body side of a constraint, the word S | base << 8 | k << 16.  Per
// iteration a body sees its hinges (by colour), then its contact normals, then the friction pairs: S = its hinges + 2 x its
// manifolds, base = the rank of this constraint's first pass in that sequence, k = its manifolds (a friction pass comes k
// after its normal pass).  Colours are unique per body, so a rank is a popcount.
B2D_D uint32_t ticket_word(uint32_t S, uint32_t base, uint32_t k) { return S | (base << 8) | (k << 16); }
B2D_D uint2 constraint_tickets(const Dev &d, uint2 pr, uint32_t col, bool hinge) {
    const unsigned long long below = (1ULL << col) - 1ULL;
    uint32_t t[2];
    const uint32_t ids[2] = {pr.x, pr.y};
    #pragma unroll
    for (int k = 0; k < 2; ++k) {
        unsigned long long bm = d.bmask[ids[k]], jm = d.jmask[ids[k]];
        uint32_t kc = __popcll(bm), kh = __popcll(jm);
        t[k] = ticket_word(kh + 2 * kc, hinge ? __popcll(jm & below) : kh + __popcll(bm & below), kc);
    }
    return make_uint2(t[0], t[1]);
}
enum PassKind { PASS_HINGE, PASS_NORMAL, PASS_FRICTION, PASS_POSITION };
struct Ticket { uint32_t ta, tb, mask; };
// The tickets a pass waits for at its two bodies.  Velocity passes: pass = iteration + 1 (0 = warm start).  Position
// passes: pass = position iteration, and as there are no friction passes a body sees S - k passes per iteration.
B2D_D uint32_t ticket_at(uint32_t w, int pass, int kind) {
    const uint32_t S = w & 0xFFu, base = (w >> 8) & 0xFFu, k = (w >> 16) & 0xFFu;
    return (uint32_t)pass * (kind == PASS_POSITION ? S - k : S) + base + (kind == PASS_FRICTION ? k : 0u);
}
B2D_D Ticket ticket_of(uint2 tk, int pass, int kind, uint32_t mask) {
    Ticket t;
    t.mask = mask; t.ta = ticket_at(tk.x, pass, kind); t.tb = ticket_at(tk.y, pass, kind);
    return t;
}

// Row preparation per sorted manifold; rows are written in colour order so the solve kernel streams them.
// k_island_tiles prepares the tiled range [0, ntiled) itself and this kernel starts after it.
__global__ void __launch_bounds__(256) k_prepare_contacts(Dev d) {
    const uint32_t n = d.cnt->nactive, first = d.cnt->ntiled;
    GRID_STRIDE(j, n - first) {
        const uint32_t i = first + j;
        uint32_t m = d.cidx_s[i];
        uint2 pr = d.mpair[m];
        uint32_t npts = d.mstate[m] & MS_NPTS_MASK;
        uint32_t fa = d.flags[pr.x], fb = d.flags[pr.y];
        SBody A = solver_body(d, pr.x, fa), B = solver_body(d, pr.y, fb);
        v3 posA = mk3(d.pos[pr.x]), posB = mk3(d.pos[pr.y]);
        q4 ornA = mkq(d.orn[pr.x]), ornB = mkq(d.orn[pr.y]);
        d.hdr[i] = make_uint4(body_tag(pr.x, A), body_tag(pr.y, B), npts,
                              slot_pair(A.proc ? d.bslot[pr.x] : SLOT_NONE, B.proc ? d.bslot[pr.y] : SLOT_NONE));
        d.tkt[i] = constraint_tickets(d, pr, (d.mstate[m] >> MS_COLOR_SHIFT) & 0xFFu, false);
        d.pisl[i] = island_of(d, pr.x, pr.y);
        for (uint32_t s = 0; s < npts; ++s) {
            const size_t ri = (size_t)s * d.NM + i;
            float4 r0, r1, r2, r3, im;
            contact_point_rows(d, (size_t)s * d.NM + m, A, B, posA, ornA, posB, ornB, r0, r1, r2, r3, im);
            d.R0[ri] = r0; d.R1[ri] = r1; d.R2[ri] = r2; d.R3[ri] = r3; d.IMP[ri] = im;
        }
    }
}

// per sorted hinge; [0, nhtiled) is prepared by k_island_tiles
__global__ void k_prepare_hinges(Dev d) {
    const uint32_t n = d.cnt->nhactive, first = d.cnt->nhtiled;
    GRID_STRIDE(j, n - first) {
        const uint32_t i = first + j;
        uint32_t h = d.hidx_s[i];
        uint2 pr = d.hpair[h];
        uint32_t fa = d.flags[pr.x], fb = d.flags[pr.y];
        SBody A = solver_body(d, pr.x, fa), B = solver_body(d, pr.y, fb);
        v3 posA = mk3(d.pos[pr.x]), posB = mk3(d.pos[pr.y]);
        q4 ornA = mkq(d.orn[pr.x]), ornB = mkq(d.orn[pr.y]);
        hinge_rows(d, h, A, B, posA, ornA, posB, ornB, d.HR + 7 * (size_t)i, 1);
        d.hhdr[i] = make_uint4(body_tag(pr.x, A), body_tag(pr.y, B), h,
                               slot_pair(A.proc ? d.bslot[pr.x] : SLOT_NONE, B.proc ? d.bslot[pr.y] : SLOT_NONE));
        d.htkt[i] = constraint_tickets(d, pr, d.hcolor[h], true);
        d.hisl[i] = island_of(d, pr.x, pr.y);
    }
}

// ====================================================================== solver: velocity iterations

// The reference sweeps the rows of an island serially (island_solver.cpp:94-111): per iteration all joint rows, all
// contact normal rows, then all friction pairs.  Here the constraints of a type are coloured so that a colour touches
// disjoint dynamic bodies; any schedule that runs a body's constraints in (iteration, type, colour) order produces the
// bits of a serial sweep in that order.  Two schedules do: k_island_tiles for small islands (everything on chip,
// __syncthreads between colours) and k_solve_df for the rest (per-body tickets in global memory).

struct VBody { v3 dv, dw; float inv_m; m3 inv_I; uint32_t id; bool proc; float pad1, pad2; };
// apply_row_impulse, constraint_row.cpp:24-32
B2D_D void apply_imp(VBody &A, VBody &B, v3 J0, v3 J1, v3 J2, v3 J3, float imp) {
    A.dv += A.inv_m * J0 * imp;
    B.dv += B.inv_m * J2 * imp;
    A.dw += A.inv_I * J1 * imp;
    B.dw += B.inv_I * J3 * imp;
}
// friction flavour keeps the reference's A-lin, A-ang, B-lin, B-ang order (constraint_row_friction.cpp:47-53)
B2D_D void apply_imp_f(VBody &A, VBody &B, v3 J0, v3 J1, v3 J2, v3 J3, float imp) {
    A.dv += A.inv_m * J0 * imp;
    A.dw += A.inv_I * J1 * imp;
    B.dv += B.inv_m * J2 * imp;
    B.dw += B.inv_I * J3 * imp;
}
// solve(constraint_row&), constraint_row.cpp:38-57
B2D_D float solve_row(float rhs, float em, float lo, float hi, float &impulse, float delta_relvel) {
    float delta = (rhs - delta_relvel) * em;
    float imp = impulse + delta;
    if (imp < lo) { delta = lo - impulse; impulse = lo; }
    else if (imp > hi) { delta = hi - impulse; impulse = hi; }
    else impulse = imp;
    return delta;
}
// one contact normal row; rows: r0 = normal | rhs, r1 = rA | eff_mass, r2 = rB | friction, im = impulses (n, t0, t1)
B2D_D void nrow_solve(const float4 &r0, const float4 &r1, const float4 &r2, float4 &im, VBody &A, VBody &B, bool warm) {
    v3 nrm = mk3(r0), rA = mk3(r1), rB = mk3(r2);
    v3 J1 = cross(rA, nrm), J2 = -nrm, J3 = -cross(rB, nrm);
    float delta;
    if (warm) delta = im.x;
    else delta = solve_row(r0.w, r1.w, 0.0f, LARGE, im.x, rel_speed(nrm, J1, J2, J3, A.dv, A.dw, B.dv, B.dw));
    apply_imp(A, B, nrm, J1, J2, J3, delta);
}
// solve_friction, constraint_row_friction.cpp:11-54: both tangent candidates from one delta-velocity snapshot,
// clamped to the circle of radius mu * lambda_n (lambda_n of THIS iteration); r3 = eff_mass t0, t1, rhs t0, t1
B2D_D void frow_solve(const float4 &r0, const float4 &r1, const float4 &r2, const float4 &r3, float4 &im, VBody &A, VBody &B, bool warm) {
    v3 nrm = mk3(r0), rA = mk3(r1), rB = mk3(r2);
    v3 t, u; plane_space(nrm, t, u);
    v3 T1 = cross(rA, t), T2 = -t, T3 = -cross(rB, t);
    v3 U1 = cross(rA, u), U2 = -u, U3 = -cross(rB, u);
    float d0, d1;
    if (warm) { d0 = im.y; d1 = im.z; }
    else {
        d0 = (r3.z - rel_speed(t, T1, T2, T3, A.dv, A.dw, B.dv, B.dw)) * r3.x;
        d1 = (r3.w - rel_speed(u, U1, U2, U3, A.dv, A.dw, B.dv, B.dw)) * r3.y;
        float i0 = im.y + d0, i1 = im.z + d1;
        float len_sqr = i0 * i0 + i1 * i1;
        float max_len = r2.w * im.x;
        if (len_sqr > max_len * max_len) {
            float len = sqrtf(len_sqr);
            if (len > EPS) { i0 = i0 / len * max_len; i1 = i1 / len * max_len; } else { i0 = 0; i1 = 0; }
            d0 = i0 - im.y; d1 = i1 - im.z;
        }
        im.y = i0; im.z = i1;
    }
    apply_imp_f(A, B, t, T1, T2, T3, d0);
    apply_imp_f(A, B, u, U1, U2, U3, d1);
}
// the five rows of a plain hinge (hinge_constraint.cpp:26-69): three point rows, two angular rows; r0..r6 as hinge_rows
// writes them, the impulses repacked into r5 / r6 (unchanged by the warm start)
B2D_D void hinge_solve(const float4 &r0, const float4 &r1, const float4 &r2, const float4 &r3, const float4 &r4, float4 &r5, float4 &r6,
                       VBody &A, VBody &B, bool warm) {
    const v3 rA = mk3(r0), rB = mk3(r1), p = mk3(r2), q = mk3(r3);
    const float em[5] = {r0.w, r1.w, r2.w, r3.w, r4.x}, rhs[5] = {r4.y, r4.z, r4.w, r5.x, r5.y};
    float imp[5] = {r5.z, r5.w, r6.x, r6.y, r6.z};
    #pragma unroll
    for (int k = 0; k < 5; ++k) {
        v3 J0, J1, J2, J3;
        if (k < 3) {
            J0 = axis_vec(k);
            v3 sa = k == 0 ? mk3(0, -rA.z, rA.y) : (k == 1 ? mk3(rA.z, 0, -rA.x) : mk3(-rA.y, rA.x, 0));
            v3 sb = k == 0 ? mk3(0, -rB.z, rB.y) : (k == 1 ? mk3(rB.z, 0, -rB.x) : mk3(-rB.y, rB.x, 0));
            J1 = -sa; J2 = -J0; J3 = sb;
        } else { v3 ax = k == 3 ? p : q; J0 = mk3(0, 0, 0); J1 = ax; J2 = mk3(0, 0, 0); J3 = -ax; }
        float delta;
        if (warm) delta = imp[k];
        else delta = solve_row(rhs[k], em[k], -SCALAR_MAX, SCALAR_MAX, imp[k], rel_speed(J0, J1, J2, J3, A.dv, A.dw, B.dv, B.dw));
        apply_imp(A, B, J0, J1, J2, J3, delta);
    }
    r5 = make_float4(r5.x, r5.y, imp[0], imp[1]); r6 = make_float4(imp[2], imp[3], imp[4], 0);
}

// ---------------------------------------------------------------------- dataflow: per-body tickets in global memory
// Instead of a grid barrier per colour, every dynamic body carries a ticket counter.  A constraint pass may touch its
// two bodies when both counters equal the tickets computed for it in k_prepare_* (position of this pass in the body's
// fixed sequence: iteration-major, then hinges / normals / frictions, then colour); afterwards it bumps them.  A pass
// waits only for its own two predecessors (an L2 round trip) rather than for the slowest CTA of the whole grid.
B2D_D void fence_gpu() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }
// ptxas recycles the unused lanes of a 128-bit load as scratch registers straight away, and the write-after-write hazard
// then parks the warp until the load has landed -- in front of the ticket poll.  keep() pins such a lane as live up to
// the point where the rest of the vector is consumed.
B2D_D void keep(float x) { asm volatile("" :: "f"(x)); }
B2D_D void keep(uint32_t x) { asm volatile("" :: "r"(x)); }
B2D_D void keep(const VBody &b) { keep(b.pad1); keep(b.pad2); }
// Dataflow acquire / publish.  The delta-velocity record of a body (two float4 = one 32 B sector) carries the
// body's ticket in BOTH .w lanes, so data and synchronisation travel in the same L2 transactions: a reader that
// sees the expected ticket in both halves has a consistent record (16 B aligned vector stores are single
// transactions; a torn pair is rejected by the double check) and needs no fence, a writer needs none either.
#ifndef B2D_LD_POLL
#define B2D_LD_POLL "ld.relaxed.gpu.global.v4.f32"     // gpu scope is all the protocol needs (.volatile = relaxed.sys)
#define B2D_ST_POLL "st.relaxed.gpu.global.v4.f32"
#endif
B2D_D float4 ld_volatile4(const float4 *p) {
    float4 v; asm volatile(B2D_LD_POLL " {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory"); return v;
}
B2D_D void st_volatile4(float4 *p, float4 v) {
    asm volatile(B2D_ST_POLL " [%0], {%1,%2,%3,%4};" :: "l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
// everything of a body that does not change during the solve
B2D_D void vb_static(const Dev &d, uint32_t tag, VBody &b) {
    b.proc = tag_proc(tag); b.id = tag_id(tag);
    b.dv = mk3(0, 0, 0); b.dw = mk3(0, 0, 0);
    if (b.proc) {
        float4 r0 = d.invIW[3 * b.id], r1 = d.invIW[3 * b.id + 1], r2 = d.invIW[3 * b.id + 2];
        b.inv_m = r0.w; b.inv_I.r0 = mk3(r0); b.inv_I.r1 = mk3(r1); b.inv_I.r2 = mk3(r2); b.pad1 = r1.w; b.pad2 = r2.w;
    } else { b.inv_m = 0; b.inv_I = m3_zero(); b.pad1 = b.pad2 = 0; }
}
B2D_D bool vb_try(const Dev &d, VBody &b, uint32_t expect) {
    float4 a = ld_volatile4(&d.dvw[2 * b.id]), w = ld_volatile4(&d.dvw[2 * b.id + 1]);
    b.dv = mk3(a); b.dw = mk3(w);
    return __float_as_uint(a.w) == expect && __float_as_uint(w.w) == expect;
}
B2D_D bool acquire_try(const Dev &d, const Ticket &t, VBody &A, VBody &B) {
    return (!A.proc || vb_try(d, A, t.ta)) & (!B.proc || vb_try(d, B, t.tb));
}
B2D_D void bodies_publish(const Dev &d, const Ticket &t, const VBody &A, const VBody &B) {
    if (A.proc) { st_volatile4(&d.dvw[2 * A.id], f4(A.dv, __uint_as_float(t.ta + 1))); st_volatile4(&d.dvw[2 * A.id + 1], f4(A.dw, __uint_as_float(t.ta + 1))); }
    if (B.proc) { st_volatile4(&d.dvw[2 * B.id], f4(B.dv, __uint_as_float(t.tb + 1))); st_volatile4(&d.dvw[2 * B.id + 1], f4(B.dw, __uint_as_float(t.tb + 1))); }
}
B2D_D bool acquire_more(const Dev &d, const Ticket &t, bool pending, bool progressed, uint32_t &spins) {
    if (!__any_sync(t.mask, pending)) return false;
    if (!__any_sync(t.mask, progressed)) {
        if (++spins > (1u << 20)) { atomicOr(&d.cnt->err, ERR_SOLVER_TIMEOUT); return false; }      // never hang the GPU
        if (spins > 64) __nanosleep(20);
    }
    return true;
}
// One pass of a constraint, for every lane of t.mask: poll() fetches the two bodies' records and says whether both carry
// the tickets of t; then work() runs and publish() writes the records with the next tickets.  Lanes of a chunk become
// ready one by one; each lane solves as soon as ITS two bodies carry the expected tickets (the ready subset runs the
// solve converged, the rest keep polling), so one late predecessor delays one constraint and not the 31 others that
// happen to share its warp.
template<typename Poll, typename Work, typename Publish>
B2D_D void ticket_wait(const Dev &d, const Ticket &t, Poll poll, Work work, Publish publish) {
    bool pending = true; uint32_t spins = 0;
    do {
        const bool ok = pending && poll();
        if (ok) {
            work();
            publish();
            pending = false;
        }
        if (!acquire_more(d, t, pending, ok, spins)) break;
    } while (true);
}

B2D_D void hinge_pass(const Dev &d, uint32_t i, bool warm, int pass, uint32_t mask) {
    uint4 hd = d.hhdr[i];
    float4 *R = d.HR + 7 * (size_t)i;
    float4 r0 = R[0], r1 = R[1], r2 = R[2], r3 = R[3], r4 = R[4], r5 = R[5], r6 = R[6];
    const Ticket tk = ticket_of(d.htkt[i], pass, PASS_HINGE, mask);
    VBody A, B; vb_static(d, hd.x, A); vb_static(d, hd.y, B);
    ticket_wait(d, tk, [&] { return acquire_try(d, tk, A, B); },
                [&] { hinge_solve(r0, r1, r2, r3, r4, r5, r6, A, B, warm); },
                [&] { bodies_publish(d, tk, A, B); if (!warm) { R[5] = r5; R[6] = r6; } });
}

// The rows of one contact point for a normal pass (NRow) or a friction pass (FRow): load() streams them in, pin() keeps
// the lanes the solve does not read, solve() runs the row and stores its impulses.
#ifndef B2D_ROW_LD
#define B2D_ROW_LD(p) __ldcs(p)       // rows stream past L1 (evict-first): the per-body data keeps it
#endif
struct NRow {
    static constexpr int KIND = PASS_NORMAL;
    float4 r0, r1, r2, im;
    B2D_D void load(const Dev &d, size_t ri) { r0 = B2D_ROW_LD(&d.R0[ri]); r1 = B2D_ROW_LD(&d.R1[ri]); r2 = B2D_ROW_LD(&d.R2[ri]); im = B2D_ROW_LD(&d.IMP[ri]); }
    B2D_D void pin() const { keep(r2.w); keep(im.y); keep(im.z); keep(im.w); }
    B2D_D void solve(const Dev &d, size_t ri, VBody &A, VBody &B, bool warm) {
        nrow_solve(r0, r1, r2, im, A, B, warm);
        if (!warm) d.IMP[ri] = im;
    }
};
struct FRow {
    static constexpr int KIND = PASS_FRICTION;
    float4 r0, r1, r2, r3, im;
    B2D_D void load(const Dev &d, size_t ri) { r0 = B2D_ROW_LD(&d.R0[ri]); r1 = B2D_ROW_LD(&d.R1[ri]); r2 = B2D_ROW_LD(&d.R2[ri]); r3 = B2D_ROW_LD(&d.R3[ri]); im = B2D_ROW_LD(&d.IMP[ri]); }
    B2D_D void pin() const { keep(r0.w); keep(r1.w); keep(im.w); }
    B2D_D void solve(const Dev &d, size_t ri, VBody &A, VBody &B, bool warm) {
        frow_solve(r0, r1, r2, r3, im, A, B, warm);
        if (!warm) d.IMP[ri] = im;
    }
};
// Row loads are issued ahead of the dependent computation: slots 0 and 1 before the ticket wait / body loads,
// slots 2 and 3 (box faces, ~15 % of manifolds) into the registers freed by slots 0 and 1 while those are being
// solved.  Impulses are private to the owning thread and stored as soon as they are final.
template<typename Row>
B2D_D void contact_pass(const Dev &d, uint32_t i, const uint4 hd, const uint2 tk2, bool warm, int pass, uint32_t mask) {
    const Ticket tk = ticket_of(tk2, pass, Row::KIND, mask);
    const uint32_t n = hd.z;
    const size_t NM = d.NM;
    Row ra, rb;
    ra.load(d, i);
    rb.load(d, n > 1 ? NM + i : i);                 // unconditional: a predicated load drags a zero-fill + WAW wait along
    VBody A, B; vb_static(d, hd.x, A); vb_static(d, hd.y, B);
    ticket_wait(d, tk, [&] { return acquire_try(d, tk, A, B); }, [&] {
        keep(A); keep(B); keep(hd.w); ra.pin(); rb.pin();
        ra.solve(d, i, A, B, warm);
        if (n > 2) ra.load(d, 2 * NM + i);
        if (n > 1) rb.solve(d, NM + i, A, B, warm);
        if (n > 3) rb.load(d, 3 * NM + i);
        if (n > 2) ra.solve(d, 2 * NM + i, A, B, warm);
        if (n > 3) rb.solve(d, 3 * NM + i, A, B, warm);
    }, [&] { bodies_publish(d, tk, A, B); });
}

// Work is dealt to warps in 32-constraint chunks that never span two colours (so lanes of a warp never wait on each
// other), chunk j to warp j mod W, each warp walking its chunks in increasing (iteration, type, colour) order.  The
// globally smallest unfinished chunk therefore always has its predecessors done and its warp working on it: no deadlock
// as long as the grid is co-resident (cooperative launch); the polls additionally bail out after a bounded number of spins.
// chunk j of a pass type -> (colour, first sorted index); `col` is a monotone cursor
B2D_D uint32_t chunk_index(const uint32_t *chunk, const uint32_t *off, uint32_t j, uint32_t &col) {
    while (j >= chunk[col + 1]) ++col;
    return off[col] + (j - chunk[col]) * 32u;
}
// colour tables of the dataflow kernels, in shared memory: every chunk walk reads them, and a global read costs an L2 round trip
struct ChunkTables { uint32_t coff[MAX_COLORS + 2], cchunk[MAX_COLORS + 2], hoff[MAX_COLORS + 2], hchunk[MAX_COLORS + 2]; };
// A warp's walk over its hinge chunks and its contact chunks.  The head of the warp's NEXT contact chunk (Head::fetch:
// header and ticket words, the same for every pass and both row types) is fetched one chunk ahead into registers, so a
// chunk starts polling its bodies without first waiting for its own header.
template<typename Head>
struct ChunkWalk {
    const ChunkTables &s;
    uint32_t lane, wid, nw, hchunks, cchunks;
    uint32_t ncol = 0, ni = 0; bool nact = false; Head next{};
    B2D_D ChunkWalk(const Dev &d, ChunkTables &t) : s(t) {
        const Counters &c = *d.cnt;
        if (threadIdx.x < MAX_COLORS + 2) {
            t.coff[threadIdx.x] = c.coff[threadIdx.x]; t.cchunk[threadIdx.x] = c.cchunk[threadIdx.x];
            t.hoff[threadIdx.x] = c.hoff[threadIdx.x]; t.hchunk[threadIdx.x] = c.hchunk[threadIdx.x];
        }
        const uint32_t nc = c.ncolors, nh = c.nhcolors;
        __syncthreads();
        lane = threadIdx.x & 31u;
        wid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; nw = (gridDim.x * blockDim.x) >> 5;
        hchunks = s.hchunk[nh]; cchunks = s.cchunk[nc];
    }
    // the head of the warp's first contact chunk
    B2D_D void start(const Dev &d) {
        if (wid < cchunks) {
            ni = chunk_index(s.cchunk, s.coff, wid, ncol) + lane; nact = ni < s.coff[ncol + 1];
            if (nact) next.fetch(d, ni);
        }
    }
    // per_lane(i, mask) for each sorted hinge i of the warp's hinge chunks
    template<typename PerLane>
    B2D_D void hinges(PerLane per_lane) {
        uint32_t col = 0;
        for (uint32_t j = wid; j < hchunks; j += nw) {
            const uint32_t i = chunk_index(s.hchunk, s.hoff, j, col) + lane;
            const bool act = i < s.hoff[col + 1];
            const uint32_t mask = __ballot_sync(0xffffffffu, act);
            if (act) per_lane(i, mask);
        }
    }
    // per_lane(i, head, mask) for each sorted manifold i of the warp's contact chunks; ahead(i, wrapped) runs once the
    // head of manifold i of the next chunk has been fetched (wrapped: that chunk is the warp's first, of the next pass)
    template<typename Ahead, typename PerLane>
    B2D_D void contacts(const Dev &d, Ahead ahead, PerLane per_lane) {
        for (uint32_t j = wid; j < cchunks; j += nw) {
            const uint32_t i = ni; const bool act = nact; const Head head = next;
            uint32_t jn = j + nw;
            if (jn >= cchunks) { jn = wid; ncol = 0; }
            ni = chunk_index(s.cchunk, s.coff, jn, ncol) + lane; nact = ni < s.coff[ncol + 1];
            if (nact) {
                next.fetch(d, ni);
                ahead(ni, jn == wid);
            }
            const uint32_t mask = __ballot_sync(0xffffffffu, act);
            if (act) per_lane(i, head, mask);
        }
    }
};
struct ContactHead {
    uint4 hd; uint2 tk;
    B2D_D void fetch(const Dev &d, uint32_t i) { hd = d.hdr[i]; tk = d.tkt[i]; }
};
B2D_D void prefetch_L2(const void *p) { asm volatile("prefetch.global.L2 [%0];" :: "l"(p)); }
#ifndef B2D_SOLVE_THREADS
#define B2D_SOLVE_THREADS 256
#endif
__global__ void __launch_bounds__(B2D_SOLVE_THREADS, 2) k_solve_df(Dev d, int iters) {
    __shared__ ChunkTables tables;
    ChunkWalk<ContactHead> walk(d, tables);
    if (walk.hchunks + walk.cchunks == 0) return;
    walk.start(d);
    for (int it = -1; it < iters; ++it) {
        const bool warm = it < 0;
        const int pass = it + 1;
        walk.hinges([&](uint32_t i, uint32_t mask) { hinge_pass(d, i, warm, pass, mask); });
        #pragma unroll 1
        for (int kind = PASS_NORMAL; kind <= PASS_FRICTION; ++kind) {
            walk.contacts(d, [&](uint32_t ni, bool wrapped) {      // the rows of the next chunk are pulled towards L2
                prefetch_L2(&d.R0[ni]); prefetch_L2(&d.R1[ni]); prefetch_L2(&d.R2[ni]); prefetch_L2(&d.IMP[ni]);
                if (kind == PASS_FRICTION || wrapped) prefetch_L2(&d.R3[ni]);
            }, [&](uint32_t i, const ContactHead &h, uint32_t mask) {
                if (kind == PASS_NORMAL) contact_pass<NRow>(d, i, h.hd, h.tk, warm, pass, mask);
                else contact_pass<FRow>(d, i, h.hd, h.tk, warm, pass, mask);
            });
        }
    }
}

// assign_applied_impulses (island_solver.cpp:232-248): rows -> warm-start cache of the constraints.
__global__ void k_store_impulses(Dev d) {
    const uint32_t n = d.cnt->nactive, nh = d.cnt->nhactive;
    const uint32_t first = d.cnt->ntiled, hfirst = d.cnt->nhtiled;       // k_island_tiles stored its own
    GRID_STRIDE(k, n - first) {
        const uint32_t i = first + k;
        const uint32_t npts = d.hdr[i].z, m = d.cidx_s[i];
        for (uint32_t s = 0; s < npts; ++s) d.pI[(size_t)s * d.NM + m] = d.IMP[(size_t)s * d.NM + i];
    }
    GRID_STRIDE(k, nh - hfirst) {
        const uint32_t i = hfirst + k;
        uint4 hd = d.hhdr[i];
        const float4 *R = d.HR + 7 * (size_t)i;
        float4 r5 = R[5], r6 = R[6];
        float *imp = d.himp + 5 * (size_t)hd.z;
        imp[0] = r5.z; imp[1] = r5.w; imp[2] = r6.x; imp[3] = r6.y; imp[4] = r6.z;
    }
}

// ====================================================================== integration and refresh

// integrate_velocities (island_solver.cpp:358-376) of one body: the delta velocities of the solve, then position and
// orientation.  Shared by k_integrate and k_island_tiles.
B2D_D void integrate_body(v3 &v, v3 &w, v3 &pos, q4 &orn, v3 dv, v3 dw, float dt) {
    v += dv; w += dw;
    pos += v * dt;
    orn = integrate(orn, w, dt);
}
// update_aabbs + update_inertias (solver.cpp:453-465) of body i at (pos, orn): the AABB of a shaped body, the world-space
// inverse inertia of a dynamic one
B2D_D void refresh_aabb(const Dev &d, uint32_t i, uint32_t f, v3 pos, q4 orn) {
    const int sk = shape_of(f);
    if (sk != SH_NONE) { box3 bb = shape_aabb(sk, d.shp[i], pos, orn); d.bbmin[i] = f4(bb.mn, 0); d.bbmax[i] = f4(bb.mx, 0); }
}
B2D_D void refresh_body(const Dev &d, uint32_t i, uint32_t f, v3 pos, q4 orn, float inv_m) {
    refresh_aabb(d, i, f, pos, orn);
    if (is_dynamic(f)) store_invIW(d, i, world_inertia(orn, load_m3(d.invI, i)), inv_m);
}
// integrate_velocities of the bodies outside the island tiles (k_island_tiles integrates and refreshes its own); with
// refresh != 0 also update_aabbs + update_inertias (solver.cpp:453-465) of them, for when no position iterations run
// in between.
__global__ void __launch_bounds__(256) k_integrate(Dev d, int refresh) {
    if (blockIdx.x == 0 && threadIdx.x == 0) d.cnt->bar = 0;       // grid barrier counter of k_position_df
    GRID_STRIDE(i, d.nbodies) {
        uint32_t f = d.flags[i];
        if (!is_dynamic(f) || d.btile[i] != TILE_NONE) continue;
        float4 p4 = d.pos[i];
        v3 pos = mk3(p4);
        q4 orn = mkq(d.orn[i]);
        v3 v = mk3(d.linvel[i]), w = mk3(d.angvel[i]);
        integrate_body(v, w, pos, orn, mk3(d.dvw[2 * i]), mk3(d.dvw[2 * i + 1]), d.dt);
        d.linvel[i] = f4(v, 0); d.angvel[i] = f4(w, 0);
        d.pos[i] = f4(pos, p4.w); d.orn[i] = f4(orn);
        d.dvw[2 * i] = make_float4(0, 0, 0, 0); d.dvw[2 * i + 1] = make_float4(0, 0, 0, 0);
        if (refresh) refresh_body(d, i, f, pos, orn, p4.w);
    }
}
// refresh_body of the dynamic and kinematic bodies after the position iterations; k_island_tiles refreshes the tiled ones
__global__ void __launch_bounds__(256) k_finalize(Dev d) {
    GRID_STRIDE(i, d.nbodies) {
        uint32_t f = d.flags[i];
        if (kind_of(f) == 2u || d.btile[i] != TILE_NONE) continue;
        float4 p4 = d.pos[i];
        refresh_body(d, i, f, mk3(p4), mkq(d.orn[i]), p4.w);
    }
}

// ====================================================================== position iterations

struct PBody { v3 pos; q4 orn; float inv_m; m3 inv_IW, inv_I; uint32_t id; bool proc; bool fresh; };   // fresh: corrected in this solve
// position_solver::solve, dynamics/position_solver.hpp:16-51.  Non-procedural bodies are left untouched
// (the reference only re-normalises their unit orientation).
B2D_D void position_solve(PBody &A, PBody &B, v3 J0, v3 J1, v3 J2, v3 J3, float error, float &max_error) {
    float s = dot(J0, J0) * A.inv_m + dot(A.inv_IW * J1, J1) + dot(J2, J2) * B.inv_m + dot(B.inv_IW * J3, J3);
    float em = 1.0f / s;
    float corr = error * 0.2f * em;
    if (A.proc) {
        A.pos += A.inv_m * J0 * corr;
        v3 ac = A.inv_IW * J1 * corr;
        A.orn = A.orn + quat_derivative(A.orn, ac);
        A.orn = normalize(A.orn);
        A.inv_IW = world_inertia(A.orn, A.inv_I); A.fresh = true;
    }
    if (B.proc) {
        B.pos += B.inv_m * J2 * corr;
        v3 ac = B.inv_IW * J3 * corr;
        B.orn = B.orn + quat_derivative(B.orn, ac);
        B.orn = normalize(B.orn);
        B.inv_IW = world_inertia(B.orn, B.inv_I); B.fresh = true;
    }
    max_error = fmaxf(fabsf(error), max_error);
}
// contact_constraint::solve_position (contact_constraint.cpp:58-90) of one contact point: refreshes its normal (pn) and
// distance (pa.w, contact_constraint.cpp:72-76), then corrects a penetration.  Shared by k_island_tiles and k_position_df;
// the latter stores the refreshed point through out_a / out_n before the correction, so fewer registers stay live across it.
B2D_D void contact_point_position(PBody &A, PBody &B, float4 &pa, const float4 &pb, float4 &pn, const float4 &pl, float &max_error,
                                  float4 *out_a = nullptr, float4 *out_n = nullptr) {
    v3 pAw = to_world(mk3(pa), A.pos, A.orn), pBw = to_world(mk3(pb), B.pos, B.orn);
    unsigned att = __float_as_uint(pl.w) & 3u;
    v3 normal = mk3(pn);
    if (att == ATT_A) normal = rotate(A.orn, mk3(pl)); else if (att == ATT_B) normal = rotate(B.orn, mk3(pl));
    float dist = dot(pAw - pBw, normal);
    v3 rA = pAw - A.pos, rB = pBw - B.pos;
    pn = f4(normal, pn.w); pa = f4(mk3(pa), dist);
    if (out_n) { *out_n = pn; *out_a = pa; }
    if (dist > -EPS) return;
    position_solve(A, B, normal, cross(rA, normal), -normal, -cross(rB, normal), -dist, max_error);
}
// hinge_constraint::solve_position, hinge_constraint.cpp:180-213; returns the max error.  Shared by k_island_tiles and
// k_position_df.
B2D_D float hinge_position(PBody &A, PBody &B, v3 fA0, v3 fB0, v3 pvA, v3 pvB) {
    float max_error = 0.0f;
    v3 axisA = rotate(A.orn, fA0), axisB = rotate(B.orn, fB0);
    v3 p, q; plane_space(axisA, p, q);
    v3 u = cross(axisA, axisB);
    const v3 z = mk3(0, 0, 0);
    { float e = dot(u, p); if (fabsf(e) > EPS) position_solve(A, B, z, p, z, -p, e, max_error); }
    { float e = dot(u, q); if (fabsf(e) > EPS) position_solve(A, B, z, q, z, -q, e, max_error); }
    v3 pivotA = to_world(pvA, A.pos, A.orn), pivotB = to_world(pvB, B.pos, B.orn);
    v3 dir = pivotA - pivotB;
    float e = length(dir);
    if (e > EPS) {
        dir /= e;
        v3 rA = pivotA - A.pos, rB = pivotB - B.pos;
        position_solve(A, B, dir, cross(rA, dir), -dir, -cross(rB, dir), -e, max_error);
    }
    return max_error;
}
// Per-island max error, aggregated per warp first: in a pile every lane belongs to the same island and one atomic per
// lane on a single address serialises the whole pass at the L2 atomic unit (0.9 ms per step at 262k bodies).
B2D_D void island_error_max(const Dev &d, uint32_t isl, float err) {
    const uint32_t active = __activemask();
    const uint32_t grp = __match_any_sync(active, isl);
    const uint32_t m = __reduce_max_sync(grp, __float_as_uint(err));
    if ((threadIdx.x & 31u) == (uint32_t)(__ffs(grp) - 1) && m) atomicMax(&d.isl_err[isl], m);
}
// the position iterations' early-out: an island whose max error fell below 0.005 is done (island_solver.cpp:538-543)
B2D_D bool island_done(float max_error) { return max_error < 0.005f; }

// per-island max error of a tile, kept at the shared-memory slot of the island's root body
B2D_D void tile_error_max(uint32_t *s_err, uint32_t islot, float err) { if (err != 0.0f) atomicMax(&s_err[islot], __float_as_uint(err)); }
// ---------------------------------------------------------------------- island tiles: the whole solver.update on chip
// row preparation + velocity iterations + integrate_velocities + assign_applied_impulses + position iterations of the
// tiled islands in ONE kernel: a tile's bodies, joints and manifolds are loaded once and their rows computed on chip, the
// velocity iterations run, the bodies are integrated
// where they sit (shared memory), the impulses go straight to the warm-start cache, the position iterations run on
// the same records, and positions / orientations / velocities are written once.  One CTA per tile; thread t owns joint t
// and manifold t of the tile for all iterations, and colours are separated by __syncthreads instead of tickets.  The row,
// solve, integration and position functions are those of the separate kernels, called in the same order
// (k_prepare_contacts, k_prepare_hinges, k_integrate, k_store_impulses, k_finalize skip what this kernel has done).  Without
// position iterations the position loop does not run and the integrated pose is written back.  Either way the AABBs and
// world-space inverse inertias of the tile's bodies are refreshed from the final pose before it leaves the CTA.
// Two specialisations of one body (island_tiles<MAXP>), by the most contact points a manifold of the tile may have:
// k_island_tiles (4) for the generic tiles, k_island_tiles_2p (2) for the two-point tiles, which keep less in registers
// (ptxas: 40 B of spills at the 128-register cap instead of 280 B; under a 3-CTA bound, 80 registers, it spilled 646 B and
// ran slower than the generic kernel on chains_1048576).  Shared memory of a tile, float4 x TILE_CAP each: body records [0..7] -- row preparation: linvel,
// angvel, inv_IW rows (| inv_m), pos, orn; velocity phase: dv, dw, inv_IW rows; position phase: pos | inv_m, orn, inv_IW
// rows, inv_I rows --, then
//   generic:   joint rows [8..14], contact points 3-4 [15..24] (solver rows, then pA pB pN pL); the solver rows of points
//              1-2 and the position-phase data of points 1-2 in registers;
//   two-point: joint rows [10..16], the solver rows of point 2 in [5..9] during the velocity iterations (body records
//              5-7 are idle then), pA pB pN pL of points 1-2 in [8..15] during the position iterations (the joint rows
//              are dead then); only the solver rows of point 1 in registers.
constexpr size_t TILE_FUSED_SMEM = (8 + 7 + 10) * TILE_CAP * sizeof(float4);
constexpr size_t TILE_FUSED_SMEM_2P = (8 + 2 + 7) * TILE_CAP * sizeof(float4);
// solver_body (+ position, orientation, record slot) of body `id` of a tiled constraint during the row preparation: a
// dynamic body from the records staged by slot, a static / kinematic one from global memory
B2D_D void tile_solver_body(const Dev &d, const float4 *sb, uint32_t id, SBody &s, v3 &pos, q4 &orn, uint32_t &slot) {
    const uint32_t f = d.flags[id];
    if (!is_dynamic(f)) { s = solver_body(d, id, f); pos = mk3(d.pos[id]); orn = mkq(d.orn[id]); slot = SLOT_NONE; return; }
    slot = d.bslot[id];
    const float4 r0 = sb[2 * TILE_CAP + slot];
    s.proc = true; s.inv_m = r0.w;
    s.inv_I.r0 = mk3(r0); s.inv_I.r1 = mk3(sb[3 * TILE_CAP + slot]); s.inv_I.r2 = mk3(sb[4 * TILE_CAP + slot]);
    s.v = mk3(sb[slot]); s.w = mk3(sb[TILE_CAP + slot]);
    pos = mk3(sb[5 * TILE_CAP + slot]); orn = mkq(sb[6 * TILE_CAP + slot]);
}
B2D_D void tf_load(const float4 *sb, uint32_t tag, uint32_t slot, VBody &b) {           // velocity phase: SoA records
    b.proc = tag_proc(tag); b.id = tag_id(tag);
    if (b.proc) {
        const float4 a = sb[slot], w = sb[TILE_CAP + slot], r0 = sb[2 * TILE_CAP + slot], r1 = sb[3 * TILE_CAP + slot], r2 = sb[4 * TILE_CAP + slot];
        b.dv = mk3(a); b.dw = mk3(w); b.inv_m = r0.w; b.inv_I.r0 = mk3(r0); b.inv_I.r1 = mk3(r1); b.inv_I.r2 = mk3(r2);
    } else { b.dv = mk3(0, 0, 0); b.dw = mk3(0, 0, 0); b.inv_m = 0; b.inv_I = m3_zero(); }
}
B2D_D void tf_store(float4 *sb, uint32_t slot, const VBody &b) {
    if (b.proc) { sb[slot] = f4(b.dv, 0); sb[TILE_CAP + slot] = f4(b.dw, 0); }
}
// position phase; a non-procedural partner (static / kinematic) is read from the thread's own copy
B2D_D void tq_load(const float4 *sb, uint32_t tag, uint32_t slot, const float4 &spos, const float4 &sorn, PBody &b) {
    b.id = tag_id(tag); b.proc = tag_proc(tag); b.fresh = false;
    if (b.proc) {
        const float4 p = sb[slot];
        b.pos = mk3(p); b.inv_m = p.w; b.orn = mkq(sb[TILE_CAP + slot]);
        b.inv_IW.r0 = mk3(sb[2 * TILE_CAP + slot]); b.inv_IW.r1 = mk3(sb[3 * TILE_CAP + slot]); b.inv_IW.r2 = mk3(sb[4 * TILE_CAP + slot]);
        b.inv_I.r0 = mk3(sb[5 * TILE_CAP + slot]); b.inv_I.r1 = mk3(sb[6 * TILE_CAP + slot]); b.inv_I.r2 = mk3(sb[7 * TILE_CAP + slot]);
    } else { b.pos = mk3(spos); b.orn = mkq(sorn); b.inv_m = 0; b.inv_IW = m3_zero(); b.inv_I = m3_zero(); }
}
B2D_D void tq_store(float4 *sb, uint32_t slot, const PBody &b) {
    if (!b.proc || !b.fresh) return;
    sb[slot] = f4(b.pos, b.inv_m); sb[TILE_CAP + slot] = f4(b.orn);
    sb[2 * TILE_CAP + slot] = f4(b.inv_IW.r0, 0); sb[3 * TILE_CAP + slot] = f4(b.inv_IW.r1, 0); sb[4 * TILE_CAP + slot] = f4(b.inv_IW.r2, 0);
}
template <int MAXP>
B2D_D void island_tiles(const Dev &d, int vel_iters, int pos_iters) {
    constexpr bool TWO = MAXP == 2;
    extern __shared__ float4 s_tile[];
    float4 *s_body = s_tile, *s_hr = s_tile + (TWO ? 10 : 8) * TILE_CAP, *s_row = s_tile + 15 * TILE_CAP;
    float4 *s_p2 = s_tile + 5 * TILE_CAP + threadIdx.x, *s_pt = s_tile + 8 * TILE_CAP + threadIdx.x;       // two-point only
    __shared__ uint32_t s_err[TILE_CAP], s_done[TILE_CAP], s_root[TILE_CAP];
    __shared__ uint32_t s_ncol[2];
    const uint32_t tile0 = TWO ? 0u : d.cnt->ntiles2, ntiles = TWO ? d.cnt->ntiles2 : d.cnt->ntiles, t = threadIdx.x;
    const size_t NM = d.NM;
    for (uint32_t tile = tile0 + blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const uint32_t nb = min(d.tile_nb[tile], (uint32_t)TILE_CAP);
        const uint32_t c0 = d.tile_c0[tile], c1 = min(d.tile_c1[tile], c0 + TILE_CAP), h0 = d.tile_h0[tile], h1 = min(d.tile_h1[tile], h0 + TILE_CAP);
        if (t < 2) s_ncol[t] = 0;
        uint32_t mybody = 0;
        if (t < nb) {       // body state for the row preparation, by slot; the velocities sit where dv, dw go until it ends
            mybody = d.tile_body[(size_t)tile * TILE_CAP + t];
            s_body[t] = d.linvel[mybody]; s_body[TILE_CAP + t] = d.angvel[mybody];
            s_body[2 * TILE_CAP + t] = d.invIW[3 * mybody]; s_body[3 * TILE_CAP + t] = d.invIW[3 * mybody + 1]; s_body[4 * TILE_CAP + t] = d.invIW[3 * mybody + 2];
            s_body[5 * TILE_CAP + t] = d.pos[mybody]; s_body[6 * TILE_CAP + t] = d.orn[mybody];
            s_err[t] = 0; s_done[t] = 0; s_root[t] = d.parent[mybody] == mybody ? 1u : 0u;
        }
        __syncthreads();
        const bool hasH = h0 + t < h1, hasC = c0 + t < c1;
        const uint32_t hi = h0 + t, ci = c0 + t;
        uint4 hh = make_uint4(0, 0, 0, 0), ch = make_uint4(0, 0, 0, 0);
        uint32_t hcol = 0xFFu, ccol = 0xFFu;
        float4 a0, a1, a2, a3, aim, b0, b1, b2, b3, bim;      // rows of contact points 1 and 2
        a0 = a1 = a2 = a3 = aim = b0 = b1 = b2 = b3 = bim = make_float4(0, 0, 0, 0);
        // ---- row preparation (k_prepare_hinges / k_prepare_contacts of the tiled range): rows go straight to where the
        // solve keeps them; hh / ch are the row headers those kernels write (tags, hinge id | point count, body slots)
        if (hasH) {
            const uint32_t h = d.hidx_s[hi];
            const uint2 pr = d.hpair[h];
            SBody A, B; v3 posA, posB; q4 ornA, ornB; uint32_t sa, sb;
            tile_solver_body(d, s_body, pr.x, A, posA, ornA, sa); tile_solver_body(d, s_body, pr.y, B, posB, ornB, sb);
            hinge_rows(d, h, A, B, posA, ornA, posB, ornB, s_hr + t, TILE_CAP);
            hh = make_uint4(body_tag(pr.x, A), body_tag(pr.y, B), h, slot_pair(sa, sb));
            hcol = d.hkey_s[hi] & 63u;
            atomicMax(&s_ncol[0], hcol + 1u);
        }
        if (hasC) {
            const uint32_t m = d.cidx_s[ci];
            const uint2 pr = d.mpair[m];
            const uint32_t npts = d.mstate[m] & MS_NPTS_MASK;
            SBody A, B; v3 posA, posB; q4 ornA, ornB; uint32_t sa, sb;
            tile_solver_body(d, s_body, pr.x, A, posA, ornA, sa); tile_solver_body(d, s_body, pr.y, B, posB, ornB, sb);
            // a two-point tile holds no manifold with more points: one that gains a third point sets graph_changed
            // (np_merge) and the rebuild moves its island to a generic tile before the next solve
            ch = make_uint4(body_tag(pr.x, A), body_tag(pr.y, B), TWO ? min(npts, 2u) : npts, slot_pair(sa, sb));
            contact_point_rows(d, m, A, B, posA, ornA, posB, ornB, a0, a1, a2, a3, aim);
            if (npts > 1) contact_point_rows(d, NM + m, A, B, posA, ornA, posB, ornB, b0, b1, b2, b3, bim);
            if (!TWO) for (uint32_t s = 2; s < npts; ++s) {
                float4 *r = s_row + (s - 2) * 5 * TILE_CAP + t;
                contact_point_rows(d, s * NM + m, A, B, posA, ornA, posB, ornB, r[0], r[TILE_CAP], r[2 * TILE_CAP], r[3 * TILE_CAP], r[4 * TILE_CAP]);
            }
            ccol = d.ckey_s[ci] & 63u;
            atomicMax(&s_ncol[1], ccol + 1u);
        }
        __syncthreads();
        if (t < nb) { s_body[t] = make_float4(0, 0, 0, 0); s_body[TILE_CAP + t] = make_float4(0, 0, 0, 0); }
        if (TWO && ch.z > 1) { s_p2[0] = b0; s_p2[TILE_CAP] = b1; s_p2[2 * TILE_CAP] = b2; s_p2[3 * TILE_CAP] = b3; s_p2[4 * TILE_CAP] = bim; }
        __syncthreads();
        const uint32_t nhc = s_ncol[0], ncc = s_ncol[1];
        // ---- velocity iterations
        for (int it = -1; it < vel_iters; ++it) {
            const bool warm = it < 0;
            for (uint32_t c = 0; c < nhc; ++c) {
                if (hcol == c) {
                    const float4 r0 = s_hr[t], r1 = s_hr[TILE_CAP + t], r2 = s_hr[2 * TILE_CAP + t], r3 = s_hr[3 * TILE_CAP + t],
                                 r4 = s_hr[4 * TILE_CAP + t];
                    float4 r5 = s_hr[5 * TILE_CAP + t], r6 = s_hr[6 * TILE_CAP + t];
                    VBody A, B; tf_load(s_body, hh.x, slot_a(hh.w), A); tf_load(s_body, hh.y, slot_b(hh.w), B);
                    hinge_solve(r0, r1, r2, r3, r4, r5, r6, A, B, warm);
                    tf_store(s_body, slot_a(hh.w), A); tf_store(s_body, slot_b(hh.w), B);
                    if (!warm) { s_hr[5 * TILE_CAP + t] = r5; s_hr[6 * TILE_CAP + t] = r6; }
                }
                __syncthreads();
            }
            for (uint32_t c = 0; c < ncc; ++c) {
                if (ccol == c) {
                    VBody A, B; tf_load(s_body, ch.x, slot_a(ch.w), A); tf_load(s_body, ch.y, slot_b(ch.w), B);
                    nrow_solve(a0, a1, a2, aim, A, B, warm);
                    if (TWO && ch.z > 1) {
                        float4 im = s_p2[4 * TILE_CAP];
                        nrow_solve(s_p2[0], s_p2[TILE_CAP], s_p2[2 * TILE_CAP], im, A, B, warm);
                        s_p2[4 * TILE_CAP] = im;
                    }
                    if (!TWO && ch.z > 1) nrow_solve(b0, b1, b2, bim, A, B, warm);
                    if (!TWO) for (uint32_t s = 2; s < ch.z; ++s) {
                        float4 *r = s_row + (s - 2) * 5 * TILE_CAP + t;
                        float4 im = r[4 * TILE_CAP];
                        nrow_solve(r[0], r[TILE_CAP], r[2 * TILE_CAP], im, A, B, warm);
                        r[4 * TILE_CAP] = im;
                    }
                    tf_store(s_body, slot_a(ch.w), A); tf_store(s_body, slot_b(ch.w), B);
                }
                __syncthreads();
            }
            for (uint32_t c = 0; c < ncc; ++c) {
                if (ccol == c) {
                    VBody A, B; tf_load(s_body, ch.x, slot_a(ch.w), A); tf_load(s_body, ch.y, slot_b(ch.w), B);
                    frow_solve(a0, a1, a2, a3, aim, A, B, warm);
                    if (TWO && ch.z > 1) {
                        float4 im = s_p2[4 * TILE_CAP];
                        frow_solve(s_p2[0], s_p2[TILE_CAP], s_p2[2 * TILE_CAP], s_p2[3 * TILE_CAP], im, A, B, warm);
                        s_p2[4 * TILE_CAP] = im;
                    }
                    if (!TWO && ch.z > 1) frow_solve(b0, b1, b2, b3, bim, A, B, warm);
                    if (!TWO) for (uint32_t s = 2; s < ch.z; ++s) {
                        float4 *r = s_row + (s - 2) * 5 * TILE_CAP + t;
                        float4 im = r[4 * TILE_CAP];
                        frow_solve(r[0], r[TILE_CAP], r[2 * TILE_CAP], r[3 * TILE_CAP], im, A, B, warm);
                        r[4 * TILE_CAP] = im;
                    }
                    tf_store(s_body, slot_a(ch.w), A); tf_store(s_body, slot_b(ch.w), B);
                }
                __syncthreads();
            }
        }
        // ---- assign_applied_impulses (k_store_impulses): rows -> warm-start cache of the constraints
        uint32_t m = 0;
        if (hasC) {
            m = d.cidx_s[ci];
            d.pI[m] = aim; if (ch.z > 1) d.pI[NM + m] = TWO ? s_p2[4 * TILE_CAP] : bim;
            if (!TWO) for (uint32_t s = 2; s < ch.z; ++s) d.pI[s * NM + m] = s_row[((s - 2) * 5 + 4) * TILE_CAP + t];
        }
        if (hasH) {
            const float4 r5 = s_hr[5 * TILE_CAP + t], r6 = s_hr[6 * TILE_CAP + t];
            float *imp = d.himp + 5 * (size_t)hh.z;
            imp[0] = r5.z; imp[1] = r5.w; imp[2] = r6.x; imp[3] = r6.y; imp[4] = r6.z;
        }
        // ---- what the position iterations need from global memory is requested before the integration below
        uint32_t hisl = 0, cisl = 0;
        v3 fA0 = mk3(0, 0, 0), fB0 = fA0, pvA = fA0, pvB = fA0;
        float4 a40, b40, n40, l40, a41, b41, n41, l41;         // contact points 1 and 2
        a40 = b40 = n40 = l40 = a41 = b41 = n41 = l41 = make_float4(0, 0, 0, 0);
        float4 spos = make_float4(0, 0, 0, 0), sorn = make_float4(0, 0, 0, 1);      // this thread's non-procedural partner (contact, else joint)
        if (hasH) {
            hisl = d.bslot[island_of(d, tag_id(hh.x), tag_id(hh.y))];
            const uint32_t h = hh.z;
            fA0 = mk3(d.hfA0[h]); fB0 = mk3(d.hfB0[h]); pvA = mk3(d.hpivA[h]); pvB = mk3(d.hpivB[h]);
        }
        if (hasC) {
            cisl = d.bslot[island_of(d, tag_id(ch.x), tag_id(ch.y))];
            if (!TWO) {
                a40 = d.pA[m]; b40 = d.pB[m]; n40 = d.pN[m]; l40 = d.pL[m];
                if (ch.z > 1) { a41 = d.pA[NM + m]; b41 = d.pB[NM + m]; n41 = d.pN[NM + m]; l41 = d.pL[NM + m]; }
            }
        }
        float4 hpos = spos, horn = sorn;                        // a joint to a static / kinematic body
        if (hasC && ((ch.x | ch.y) >> 31)) { const uint32_t sbody = tag_id(tag_proc(ch.x) ? ch.y : ch.x); spos = d.pos[sbody]; sorn = d.orn[sbody]; }
        if (hasH && ((hh.x | hh.y) >> 31)) { const uint32_t sbody = tag_id(tag_proc(hh.x) ? hh.y : hh.x); hpos = d.pos[sbody]; horn = d.orn[sbody]; }
        __syncthreads();                                         // the rows in s_row (two-point: s_p2, s_hr) are dead from here on
        if (hasC) for (uint32_t s = TWO ? 0 : 2; s < ch.z; ++s) {
            const size_t mi = s * NM + m;
            float4 *r = TWO ? s_pt + s * 4 * TILE_CAP : s_row + (s - 2) * 4 * TILE_CAP + t;
            r[0] = d.pA[mi]; r[TILE_CAP] = d.pB[mi]; r[2 * TILE_CAP] = d.pN[mi]; r[3 * TILE_CAP] = d.pL[mi];
        }
        // ---- integrate_velocities (k_integrate) for the tile's bodies; the records turn into position records
        if (t < nb) {
            v3 v = mk3(d.linvel[mybody]), w = mk3(d.angvel[mybody]), pos = mk3(d.pos[mybody]);
            q4 orn = mkq(d.orn[mybody]);
            integrate_body(v, w, pos, orn, mk3(s_body[t]), mk3(s_body[TILE_CAP + t]), d.dt);
            d.linvel[mybody] = f4(v, 0); d.angvel[mybody] = f4(w, 0);
            s_body[t] = f4(pos, s_body[2 * TILE_CAP + t].w);     // inverse mass as the solvers see it
            s_body[TILE_CAP + t] = f4(orn);
            s_body[5 * TILE_CAP + t] = d.invI[3 * mybody]; s_body[6 * TILE_CAP + t] = d.invI[3 * mybody + 1]; s_body[7 * TILE_CAP + t] = d.invI[3 * mybody + 2];
        }
        __syncthreads();
        // ---- position iterations: <= N, each island stopping once island_done (island_solver.cpp:263-353); per-island error / done words sit at the slot of the island's root body; the contact points of the first two
        // slots stay in registers, their refreshed normal and distance (contact_constraint.cpp:72-76) are written back at the end
        for (int it = 0; it < pos_iters; ++it) {
            for (uint32_t c = 0; c < nhc; ++c) {
                if (hcol == c && !s_done[hisl]) {
                    PBody A, B; tq_load(s_body, hh.x, slot_a(hh.w), hpos, horn, A); tq_load(s_body, hh.y, slot_b(hh.w), hpos, horn, B);
                    const float max_error = hinge_position(A, B, fA0, fB0, pvA, pvB);
                    tq_store(s_body, slot_a(hh.w), A); tq_store(s_body, slot_b(hh.w), B);
                    tile_error_max(s_err, hisl, max_error);
                }
                __syncthreads();
            }
            for (uint32_t c = 0; c < ncc; ++c) {
                if (ccol == c && !s_done[cisl]) {
                    PBody A, B; tq_load(s_body, ch.x, slot_a(ch.w), spos, sorn, A); tq_load(s_body, ch.y, slot_b(ch.w), spos, sorn, B);
                    float max_error = 0.0f;
                    if (!TWO) {
                        contact_point_position(A, B, a40, b40, n40, l40, max_error);
                        if (ch.z > 1) contact_point_position(A, B, a41, b41, n41, l41, max_error);
                    }
                    for (uint32_t s = TWO ? 0 : 2; s < ch.z; ++s) {
                        float4 *r = TWO ? s_pt + s * 4 * TILE_CAP : s_row + (s - 2) * 4 * TILE_CAP + t;
                        float4 pa = r[0], pn = r[2 * TILE_CAP];
                        contact_point_position(A, B, pa, r[TILE_CAP], pn, r[3 * TILE_CAP], max_error);
                        r[0] = pa; r[2 * TILE_CAP] = pn;
                    }
                    tq_store(s_body, slot_a(ch.w), A); tq_store(s_body, slot_b(ch.w), B);
                    tile_error_max(s_err, cisl, max_error);
                }
                __syncthreads();
            }
            if (it + 1 < pos_iters) {
                if (t < nb && s_root[t]) { if (island_done(__uint_as_float(s_err[t]))) s_done[t] = 1; s_err[t] = 0; }
                __syncthreads();
            }
        }
        if (hasC) {
            if (!TWO) {
                d.pN[m] = n40; d.pA[m] = a40;
                if (ch.z > 1) { d.pN[NM + m] = n41; d.pA[NM + m] = a41; }
            }
            for (uint32_t s = TWO ? 0 : 2; s < ch.z; ++s) {
                const float4 *r = TWO ? s_pt + s * 4 * TILE_CAP : s_row + (s - 2) * 4 * TILE_CAP + t;
                d.pA[s * NM + m] = r[0]; d.pN[s * NM + m] = r[2 * TILE_CAP];
            }
        }
        // the final pose, then update_aabbs + update_inertias of it (k_finalize and k_integrate skip tiled bodies), with
        // inv_I from records 5-7; the body id is read again from the tile list rather than held across the iterations
        if (t < nb) {
            const uint32_t i = d.tile_body[(size_t)tile * TILE_CAP + t];
            const float4 p = s_body[t], o = s_body[TILE_CAP + t];
            const float inv_m = d.pos[i].w;
            d.pos[i] = make_float4(p.x, p.y, p.z, inv_m); d.orn[i] = o;
            m3 inv_I; inv_I.r0 = mk3(s_body[5 * TILE_CAP + t]); inv_I.r1 = mk3(s_body[6 * TILE_CAP + t]); inv_I.r2 = mk3(s_body[7 * TILE_CAP + t]);
            refresh_aabb(d, i, d.flags[i], mk3(p), mkq(o));             // a tiled body is dynamic
            store_invIW(d, i, world_inertia(mkq(o), inv_I), inv_m);
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(TILE_CAP, 2) k_island_tiles(Dev d, int vel_iters, int pos_iters) { island_tiles<4>(d, vel_iters, pos_iters); }
__global__ void __launch_bounds__(TILE_CAP, 2) k_island_tiles_2p(Dev d, int vel_iters, int pos_iters) { island_tiles<2>(d, vel_iters, pos_iters); }

// ---------------------------------------------------------------------- dataflow: position iterations
#ifndef B2D_POS_MIN_BLOCKS
#define B2D_POS_MIN_BLOCKS 1
#endif
#ifndef B2D_POS_THREADS
#define B2D_POS_THREADS 256
#endif

// ---- dataflow flavour of the position iterations (default).  Same idea as k_solve_df: what a constraint needs from a
// body AND the body's ticket travel in the same 16-byte vectors, so a poll that sees the expected ticket in all three
// vectors of a record already holds a consistent position / orientation and no fence or separate counter is needed.
// The record does not carry the world-space inverse inertia: a body that was corrected at least once in this solve
// ("fresh") has inv_IW == world_inertia(orn, inv_I) exactly (position_solve recomputes it that way), so the reader
// recomputes it from the orientation; an untouched body still uses the tensor of the previous step (the reference
// refreshes inertia only after the position iterations, solver.cpp:453-465), read from d.invIW.
struct PRec { float4 p0, p1, p2; };
B2D_D void prec_issue(const Dev &d, uint32_t id, PRec &r) {
    const float4 *p = d.prec + 3 * (size_t)id;
    r.p0 = ld_volatile4(p); r.p1 = ld_volatile4(p + 1); r.p2 = ld_volatile4(p + 2);
}
B2D_D bool prec_ok(const PRec &r, uint32_t t) {
    return __float_as_uint(r.p0.w) == t && __float_as_uint(r.p1.w) == t && __float_as_uint(r.p2.w) == t;
}
B2D_D void prec_take(const PRec &r, PBody &b, const m3 &stale) {
    b.pos = mk3(r.p0); b.orn.x = r.p1.x; b.orn.y = r.p1.y; b.orn.z = r.p1.z; b.orn.w = r.p2.x;
    b.fresh = r.p2.y != 0.0f;
    b.inv_IW = b.fresh ? world_inertia(b.orn, b.inv_I) : stale;
}
B2D_D void prec_publish(const Dev &d, const PBody &b, uint32_t t) {
    float4 *p = d.prec + 3 * (size_t)b.id;
    const float tf = __uint_as_float(t);
    st_volatile4(p, f4(b.pos, tf)); st_volatile4(p + 1, make_float4(b.orn.x, b.orn.y, b.orn.z, tf)); st_volatile4(p + 2, make_float4(b.orn.w, b.fresh ? 1.0f : 0.0f, 0.0f, tf));
}
// everything of a body that does not change during the solve; `stale` = inverse world inertia of the previous step
B2D_D void pb_begin(const Dev &d, uint32_t id, bool proc, PBody &b, m3 &stale) {
    b.id = id; b.proc = proc; b.fresh = false;
    if (proc) {
        const float4 r0 = d.invIW[3 * id], r1 = d.invIW[3 * id + 1], r2 = d.invIW[3 * id + 2];
        b.inv_m = r0.w; stale.r0 = mk3(r0); stale.r1 = mk3(r1); stale.r2 = mk3(r2);
        b.inv_I = load_m3(d.invI, id);
    } else {
        b.pos = mk3(d.pos[id]); b.orn = mkq(d.orn[id]);
        b.inv_m = 0; b.inv_IW = m3_zero(); b.inv_I = m3_zero(); stale = m3_zero();
    }
}
// One chunk of position constraints.  `work` runs the constraint on (A, B) and returns its max error.
template<typename Work>
B2D_D void position_chunk_df(const Dev &d, uint32_t tagA, uint32_t tagB, uint2 tk2, uint32_t isl, int it, uint32_t mask, Work work) {
    const uint32_t a = tag_id(tagA), b = tag_id(tagB);
    const bool pa = tag_proc(tagA), pb = tag_proc(tagB);
    // all constraints of a finished island skip together (and keep skipping), so their tickets stay consistent
    const bool skip = __ldcg(&d.isl_done[isl]) != 0;
    PBody A, B; m3 staleA, staleB;
    pb_begin(d, a, pa, A, staleA); pb_begin(d, b, pb, B, staleB);
    const uint32_t live = __ballot_sync(mask, !skip);
    if (skip) return;
    const Ticket tk = ticket_of(tk2, it, PASS_POSITION, live);
    // ticket_wait's loop, written out: through the template k_position_df needs 2 more registers (ptxas, sm_90a).  Unlike
    // ticket_wait it polls whether or not the lane is pending; a lane that is done finds its bodies past its tickets.
    bool pending = true; uint32_t spins = 0;
    do {
        PRec ra, rb;
        if (pa) prec_issue(d, a, ra);
        if (pb) prec_issue(d, b, rb);
        const bool ok = (!pa || prec_ok(ra, tk.ta)) & (!pb || prec_ok(rb, tk.tb));
        if (ok) {
            if (pa) prec_take(ra, A, staleA);
            if (pb) prec_take(rb, B, staleB);
            const float max_error = work(A, B);
            if (pa) prec_publish(d, A, tk.ta + 1);
            if (pb) prec_publish(d, B, tk.tb + 1);
            island_error_max(d, isl, max_error);
            pending = false;
        }
        if (!acquire_more(d, tk, pending, ok, spins)) break;
    } while (true);
}
// contact_constraint::solve_position, contact_constraint.cpp:58-90
B2D_D void contact_position_df(const Dev &d, uint4 hd, uint32_t m, uint2 tk2, uint32_t isl, int it, uint32_t mask) {
    const uint32_t n = hd.z;
    const size_t NM = d.NM;
    // slot 0 of the manifold is in flight while the tickets are polled
    const float4 a0 = d.pA[m], b0 = d.pB[m], n0 = d.pN[m], l0 = d.pL[m];
    position_chunk_df(d, hd.x, hd.y, tk2, isl, it, mask, [&](PBody &A, PBody &B) {
        float max_error = 0.0f;
        float4 a4 = a0, b4 = b0, n4 = n0, l4 = l0;
        for (uint32_t s = 0; s < n; ++s) {
            const size_t mi = (size_t)s * NM + m;
            if (s) { a4 = d.pA[mi]; b4 = d.pB[mi]; n4 = d.pN[mi]; l4 = d.pL[mi]; }
            contact_point_position(A, B, a4, b4, n4, l4, max_error, &d.pA[mi], &d.pN[mi]);
        }
        return max_error;
    });
}
B2D_D void hinge_position_df(const Dev &d, uint4 hd, uint2 tk2, uint32_t isl, int it, uint32_t mask) {
    const uint32_t h = hd.z;
    const v3 fA0 = mk3(d.hfA0[h]), fB0 = mk3(d.hfB0[h]), pvA = mk3(d.hpivA[h]), pvB = mk3(d.hpivB[h]);
    position_chunk_df(d, hd.x, hd.y, tk2, isl, it, mask, [&](PBody &A, PBody &B) { return hinge_position(A, B, fA0, fB0, pvA, pvB); });
}
// what the position iterations fetch one chunk ahead: also the island label and the manifold slot
struct PositionHead {
    uint4 hd; uint2 tk; uint32_t isl, m;
    B2D_D void fetch(const Dev &d, uint32_t i) { hd = d.hdr[i]; tk = d.tkt[i]; isl = d.pisl[i]; m = d.cidx_s[i]; }
};
__global__ void __launch_bounds__(B2D_POS_THREADS, B2D_POS_MIN_BLOCKS) k_position_df(Dev d, int iters) {
    __shared__ ChunkTables tables;
    GridBarrier grid(&d.cnt->bar);
    ChunkWalk<PositionHead> walk(d, tables);
    if (walk.hchunks + walk.cchunks == 0) return;       // every island is tiled (the whole grid takes this exit together)
    GRID_STRIDE(i, d.nbodies) {
        d.isl_err[i] = 0; d.isl_done[i] = 0;
        if (is_dynamic(d.flags[i])) {
            const float4 p4 = d.pos[i], o4 = d.orn[i];
            float4 *r = d.prec + 3 * (size_t)i;
            r[0] = make_float4(p4.x, p4.y, p4.z, 0.0f); r[1] = make_float4(o4.x, o4.y, o4.z, 0.0f); r[2] = make_float4(o4.w, 0.0f, 0.0f, 0.0f);
        }
    }
    walk.start(d);
    grid.sync();
    for (int it = 0; it < iters; ++it) {
        walk.hinges([&](uint32_t i, uint32_t mask) { hinge_position_df(d, d.hhdr[i], d.htkt[i], d.hisl[i], it, mask); });
        walk.contacts(d, [](uint32_t, bool) {}, [&](uint32_t, const PositionHead &h, uint32_t mask) {
            contact_position_df(d, h.hd, h.m, h.tk, h.isl, it, mask);
        });
        if (it + 1 < iters) {
            grid.sync();
            GRID_STRIDE(i, d.nbodies) {
                if (d.parent[i] == i) { if (island_done(__uint_as_float(d.isl_err[i]))) d.isl_done[i] = 1; d.isl_err[i] = 0; }
            }
            grid.sync();
        }
    }
    grid.sync();
    GRID_STRIDE(i, d.nbodies) {
        if (is_dynamic(d.flags[i])) {
            const float4 *r = d.prec + 3 * (size_t)i;
            const float4 r0 = __ldcg(r), r1 = __ldcg(r + 1), r2 = __ldcg(r + 2);
            if (r2.y != 0.0f) {        // corrected at least once
                d.pos[i] = make_float4(r0.x, r0.y, r0.z, d.pos[i].w); d.orn[i] = make_float4(r1.x, r1.y, r1.z, r2.x);
            }
        }
    }
}

// ====================================================================== multi-GPU: bounds of the owned islands

// Bounding box of every dynamic body's AABB, reduced on the device into a caller-provided DEVICE buffer of 6 floats
// (min xyz, max xyz) that the host adapter all-gathers over NCCL: the cross-GPU AABB-overlap exchange of SURVEY 8e at
// rank granularity.  Floats are compared through an order-preserving int encoding so plain atomicMin/Max work.
B2D_D int f2ord(float f) { int i = __float_as_int(f); return i >= 0 ? i : i ^ 0x7FFFFFFF; }
B2D_D float ord2f(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7FFFFFFF); }
__global__ void k_bounds_init(Dev d) {
    if (blockIdx.x == 0 && threadIdx.x < 6) d.cnt->bounds[threadIdx.x] = threadIdx.x < 3 ? f2ord(INFINITY) : f2ord(-INFINITY);
    if (blockIdx.x == 0 && threadIdx.x == 6) d.cnt->speed = 0;
}
// + the largest distance any point of any body can travel per second at its current velocity (|v| + |w| r, r = half
// diagonal of the AABB): lets the host look one step ahead when it overlaps the exchange with the next step
__global__ void k_bounds_reduce(Dev d) {
    float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY}, sp = 0.0f;
    GRID_STRIDE(i, d.nbodies) {
        uint32_t f = d.flags[i];
        if (!is_procedural(f) || shape_of(f) == SH_NONE) continue;
        float4 a = d.bbmin[i], b = d.bbmax[i];
        mn[0] = fminf(mn[0], a.x); mn[1] = fminf(mn[1], a.y); mn[2] = fminf(mn[2], a.z);
        mx[0] = fmaxf(mx[0], b.x); mx[1] = fmaxf(mx[1], b.y); mx[2] = fmaxf(mx[2], b.z);
        if (is_dynamic(f)) sp = fmaxf(sp, length(mk3(d.linvel[i])) + length(mk3(d.angvel[i])) * 0.5f * length(mk3(b) - mk3(a)));
    }
    #pragma unroll
    for (int k = 0; k < 3; ++k) {
        for (int o = 16; o > 0; o >>= 1) { mn[k] = fminf(mn[k], __shfl_xor_sync(0xffffffffu, mn[k], o)); mx[k] = fmaxf(mx[k], __shfl_xor_sync(0xffffffffu, mx[k], o)); }
        if ((threadIdx.x & 31) == 0) { atomicMin(&d.cnt->bounds[k], f2ord(mn[k])); atomicMax(&d.cnt->bounds[3 + k], f2ord(mx[k])); }
    }
    for (int o = 16; o > 0; o >>= 1) sp = fmaxf(sp, __shfl_xor_sync(0xffffffffu, sp, o));
    if ((threadIdx.x & 31) == 0 && sp > 0.0f) atomicMax(&d.cnt->speed, __float_as_uint(sp));      // non-negative floats order like their bits
}
__global__ void k_bounds_final(Dev d, float *out8) {
    if (blockIdx.x == 0 && threadIdx.x < 6) out8[threadIdx.x] = ord2f(d.cnt->bounds[threadIdx.x]);
    if (blockIdx.x == 0 && threadIdx.x == 6) { out8[6] = __uint_as_float(d.cnt->speed); out8[7] = 0.0f; }
}

// ====================================================================== statistics
__global__ void k_count_points(Dev d) {
    const uint32_t hwm = d.cnt->hwm;
    uint32_t local = 0;
    GRID_STRIDE(m, hwm) { uint32_t st = d.mstate[m]; if (st & MS_ALIVE) local += st & MS_NPTS_MASK; }
    for (int o = 16; o > 0; o >>= 1) local += __shfl_down_sync(0xffffffffu, local, o);
    if ((threadIdx.x & 31) == 0 && local) atomicAdd(&d.cnt->npoints, local);
}

// ====================================================================== restitution solver
// dynamics/restitution_solver.cpp:86-408 (settings: 8 rounds x 3 sweeps by default).  Before gravity is applied, per island
// and per round: the manifold with contact_manifold_with_restitution that closes fastest; if it closes faster than 0.005 m/s,
// a breadth-first walk of the entity graph from the faster of its two bodies; at every dynamic body visited, the manifolds
// of that body still closing faster than the threshold are solved together -- rows from the CURRENT velocities with the
// points' restitution, a few Gauss-Seidel sweeps (normal row, then its friction pair), then the delta velocities are added
// to the velocities at once.  Afterwards the ordinary rows carry no restitution (solver.cpp:217-236).
// The walk is serial by construction, so is this: ONE THREAD PER ISLAND (islands are independent; a scene of many small
// islands parallelises over them, a single pile does not -- DESIGN.md section 8).  Orders the reference takes from EnTT and
// the graph's history are fixed here: neighbours in ascending body id, ties of the fastest manifold to the smaller pair key.
constexpr int REST_MAX_MANIFOLDS = 32;      // manifolds of one body solved as a group
constexpr int REST_MAX_ROWS = 96;           // their contact points

// the entity graph as adjacency lists: manifolds (with or without points) and joints are edges
__global__ void k_rest_count(Dev d) {
    const uint32_t hwm = d.cnt->hwm;
    GRID_STRIDE(k, hwm + d.nhinges) {
        uint2 p;
        if (k < hwm) { if (!(d.mstate[k] & MS_ALIVE)) continue; p = d.mpair[k]; }
        else { p = d.hpair[k - hwm]; if (p.x == p.y) continue; }
        if (is_dynamic(d.flags[p.x])) atomicAdd(&d.rcnt[p.x], 1u);
        if (is_dynamic(d.flags[p.y])) atomicAdd(&d.rcnt[p.y], 1u);
    }
}
__global__ void k_rest_fill(Dev d) {
    const uint32_t hwm = d.cnt->hwm;
    GRID_STRIDE(k, hwm + d.nhinges) {
        uint2 p; uint32_t tag = 0, slot = 0;
        if (k < hwm) { if (!(d.mstate[k] & MS_ALIVE)) continue; p = d.mpair[k]; tag = 0x80000000u; slot = k; }
        else { p = d.hpair[k - hwm]; if (p.x == p.y) continue; }
        if (is_dynamic(d.flags[p.x])) { const uint32_t at = d.roff[p.x] + atomicAdd(&d.rcur[p.x], 1u); d.radj[at] = p.y | tag; d.radj_m[at] = slot; }
        if (is_dynamic(d.flags[p.y])) { const uint32_t at = d.roff[p.y] + atomicAdd(&d.rcur[p.y], 1u); d.radj[at] = p.x | tag; d.radj_m[at] = slot; }
    }
}
// ascending neighbour id, one entry per neighbour (a joint and a manifold between the same two bodies share an adjacency)
__global__ void k_rest_sort(Dev d) {
    GRID_STRIDE(b, d.nbodies) {
        const uint32_t n = d.rcnt[b], o = d.roff[b];
        if (n == 0) continue;
        for (uint32_t i = 1; i < n; ++i) {
            const uint32_t e = d.radj[o + i], m = d.radj_m[o + i];
            uint32_t j = i;
            while (j > 0 && (d.radj[o + j - 1] & 0x7FFFFFFFu) > (e & 0x7FFFFFFFu)) { d.radj[o + j] = d.radj[o + j - 1]; d.radj_m[o + j] = d.radj_m[o + j - 1]; --j; }
            d.radj[o + j] = e; d.radj_m[o + j] = m;
        }
        uint32_t w = 0;
        for (uint32_t i = 0; i < n; ++i) {
            const uint32_t e = d.radj[o + i], m = d.radj_m[o + i];
            if (w && (d.radj[o + w - 1] & 0x7FFFFFFFu) == (e & 0x7FFFFFFFu)) { if (e >> 31) { d.radj[o + w - 1] |= 0x80000000u; d.radj_m[o + w - 1] = m; } }
            else { d.radj[o + w] = e; d.radj_m[o + w] = m; ++w; }
        }
        d.rcnt[b] = w;
    }
}
// get_manifold_min_relvel, restitution_solver.cpp:32-83
B2D_D float rest_min_relvel(const Dev &d, uint32_t m) {
    const uint2 pr = d.mpair[m];
    const uint32_t npts = d.mstate[m] & MS_NPTS_MASK;
    const uint32_t fa = d.flags[pr.x], fb = d.flags[pr.y];
    const v3 z = mk3(0, 0, 0);
    const v3 lvA = kind_of(fa) == 2u ? z : mk3(d.linvel[pr.x]), avA = kind_of(fa) == 2u ? z : mk3(d.angvel[pr.x]);
    const v3 lvB = kind_of(fb) == 2u ? z : mk3(d.linvel[pr.y]), avB = kind_of(fb) == 2u ? z : mk3(d.angvel[pr.y]);
    const v3 posA = mk3(d.pos[pr.x]), posB = mk3(d.pos[pr.y]);
    const q4 ornA = mkq(d.orn[pr.x]), ornB = mkq(d.orn[pr.y]);
    float min_relvel = SCALAR_MAX;
    for (uint32_t s = 0; s < npts; ++s) {
        const size_t mi = (size_t)s * d.NM + m;
        const v3 pivotA = to_world(mk3(d.pA[mi]), posA, ornA), pivotB = to_world(mk3(d.pB[mi]), posB, ornB);
        const v3 rA = pivotA - posA, rB = pivotB - posB;
        const v3 vA = lvA + cross(avA, rA), vB = lvB + cross(avB, rB);
        const v3 relvel = vA - vB;
        min_relvel = fminf(dot(relvel, mk3(d.pN[mi])), min_relvel);
    }
    return min_relvel;
}
B2D_D void rest_body_load(const Dev &d, uint32_t i, VBody &b) {
    b.id = i; b.proc = is_dynamic(d.flags[i]);
    if (b.proc) {
        const float4 r0 = d.invIW[3 * i];
        b.inv_m = r0.w; b.inv_I.r0 = mk3(r0); b.inv_I.r1 = mk3(d.invIW[3 * i + 1]); b.inv_I.r2 = mk3(d.invIW[3 * i + 2]);
        b.dv = mk3(d.dvw[2 * i]); b.dw = mk3(d.dvw[2 * i + 1]);
    } else { b.inv_m = 0; b.inv_I = m3_zero(); b.dv = mk3(0, 0, 0); b.dw = mk3(0, 0, 0); }
}
B2D_D void rest_body_store(const Dev &d, const VBody &b) {
    if (b.proc) { d.dvw[2 * b.id] = f4(b.dv, 0.0f); d.dvw[2 * b.id + 1] = f4(b.dw, 0.0f); }
}
// the solve_manifolds lambda, restitution_solver.cpp:146-310
B2D_D void rest_solve_group(const Dev &d, const uint32_t *group, int ng) {
    float4 r0[REST_MAX_ROWS], r1[REST_MAX_ROWS], r2[REST_MAX_ROWS], r3[REST_MAX_ROWS], im[REST_MAX_ROWS];
    uint32_t ra[REST_MAX_ROWS], rb[REST_MAX_ROWS];
    int nr = 0;
    for (int g = 0; g < ng; ++g) {
        const uint32_t m = group[g];
        const uint2 pr = d.mpair[m];
        const uint32_t npts = d.mstate[m] & MS_NPTS_MASK;
        const SBody A = solver_body(d, pr.x, d.flags[pr.x]), B = solver_body(d, pr.y, d.flags[pr.y]);
        const v3 posA = mk3(d.pos[pr.x]), posB = mk3(d.pos[pr.y]);
        const q4 ornA = mkq(d.orn[pr.x]), ornB = mkq(d.orn[pr.y]);
        for (uint32_t s = 0; s < npts; ++s) {
            if (nr == REST_MAX_ROWS) { atomicOr(&d.cnt->err, ERR_RESTITUTION_GROUP); break; }
            contact_point_rows(d, (size_t)s * d.NM + m, A, B, posA, ornA, posB, ornB, r0[nr], r1[nr], r2[nr], r3[nr], im[nr], true);
            ra[nr] = pr.x; rb[nr] = pr.y;
            ++nr;
        }
    }
    for (uint32_t it = 0; it < d.rest_individual; ++it) {
        for (int k = 0; k < nr; ++k) {
            VBody A, B;
            rest_body_load(d, ra[k], A); rest_body_load(d, rb[k], B);
            nrow_solve(r0[k], r1[k], r2[k], im[k], A, B, false);
            frow_solve(r0[k], r1[k], r2[k], r3[k], im[k], A, B, false);
            rest_body_store(d, A); rest_body_store(d, B);
        }
    }
    for (int g = 0; g < ng; ++g) {                             // apply the delta velocities (idempotent for shared bodies)
        const uint2 pr = d.mpair[group[g]];
        const uint32_t ids[2] = {pr.x, pr.y};
        for (int k = 0; k < 2; ++k) {
            const uint32_t i = ids[k];
            if (!is_dynamic(d.flags[i])) continue;                 // static: skipped; kinematic: its deltas are the dummy zeros
            d.linvel[i] = f4(mk3(d.linvel[i]) + mk3(d.dvw[2 * i]), 0.0f);
            d.angvel[i] = f4(mk3(d.angvel[i]) + mk3(d.dvw[2 * i + 1]), 0.0f);
            d.dvw[2 * i] = make_float4(0, 0, 0, 0); d.dvw[2 * i + 1] = make_float4(0, 0, 0, 0);
        }
    }
}
__global__ void k_rest_solve(Dev d) {
    constexpr uint32_t NONE = 0xFFFFFFFFu;
    const float threshold = -0.005f;
    GRID_STRIDE(root, d.nbodies) {
        if (d.parent[root] != root || !is_dynamic(d.flags[root])) continue;       // one thread per awake island
        uint32_t stamp = 0;
        for (uint32_t round = 0; round < d.rest_iters; ++round) {
            // ---- the manifold with restitution that closes fastest (walk over the island)
            float best = SCALAR_MAX; uint32_t best_m = NONE; unsigned long long best_key = ~0ULL;
            ++stamp;
            uint32_t head = root, tail = root;
            d.rstamp[root] = stamp; d.rnext[root] = NONE;
            while (head != NONE) {
                const uint32_t b = head; head = d.rnext[b];
                const uint32_t o = d.roff[b], n = d.rcnt[b];
                for (uint32_t k = 0; k < n; ++k) {
                    const uint32_t e = d.radj[o + k], nbr = e & 0x7FFFFFFFu;
                    if (e >> 31) {
                        const uint32_t m = d.radj_m[o + k];
                        const uint2 pr = d.mpair[m];
                        if (fminf(d.mat[pr.x].y, d.mat[pr.y].y) > EPS) {            // contact_manifold_with_restitution, constraint_util.cpp:86-101
                            const float rel = rest_min_relvel(d, m);
                            const unsigned long long key = pair_key(pr.x, pr.y);
                            if (rel < best || (rel == best && best_m != NONE && key < best_key)) { best = rel; best_m = m; best_key = key; }
                        }
                    }
                    if (is_dynamic(d.flags[nbr]) && d.rstamp[nbr] != stamp) {
                        d.rstamp[nbr] = stamp; d.rnext[nbr] = NONE;
                        if (head == NONE) head = nbr; else d.rnext[tail] = nbr;
                        tail = nbr;
                    }
                }
            }
            if (best_m == NONE || best > threshold) break;                          // nothing (left) to bounce in this island
            // ---- start at the faster body of that manifold (a dynamic one)
            const uint2 fp = d.mpair[best_m];
            const uint32_t fa = d.flags[fp.x], fb = d.flags[fp.y];
            const float speedA = kind_of(fa) == 2u ? 0.0f : length_sqr(mk3(d.linvel[fp.x]));
            const float speedB = kind_of(fb) == 2u ? 0.0f : length_sqr(mk3(d.linvel[fp.y]));
            uint32_t start;
            if (speedA > speedB) start = is_dynamic(fa) ? fp.x : fp.y; else start = is_dynamic(fb) ? fp.y : fp.x;
            // ---- breadth-first: at every body the manifolds still closing fast enough, solved as a group
            ++stamp;
            head = start; tail = start;
            d.rstamp[start] = stamp; d.rnext[start] = NONE;
            while (head != NONE) {
                const uint32_t b = head; head = d.rnext[b];
                const uint32_t o = d.roff[b], n = d.rcnt[b];
                uint32_t group[REST_MAX_MANIFOLDS]; int ng = 0;
                for (uint32_t k = 0; k < n; ++k) {
                    if (!(d.radj[o + k] >> 31)) continue;
                    const uint32_t m = d.radj_m[o + k];
                    if (rest_min_relvel(d, m) < threshold) {
                        if (ng == REST_MAX_MANIFOLDS) { atomicOr(&d.cnt->err, ERR_RESTITUTION_GROUP); break; }
                        group[ng++] = m;
                    }
                }
                if (ng) rest_solve_group(d, group, ng);
                for (uint32_t k = 0; k < n; ++k) {
                    const uint32_t nbr = d.radj[o + k] & 0x7FFFFFFFu;
                    if (is_dynamic(d.flags[nbr]) && d.rstamp[nbr] != stamp) {
                        d.rstamp[nbr] = stamp; d.rnext[nbr] = NONE;
                        if (head == NONE) head = nbr; else d.rnext[tail] = nbr;
                        tail = nbr;
                    }
                }
            }
        }
    }
}

// ====================================================================== raycast (edyn::raycast, src/edyn/collision/raycast.cpp:20-56)
// Batched segment queries against the current AABBs (DESIGN.md §2b).  The index is the broadphase's uniform grid
// rebuilt into buffers of its own: bodies are binned by AABB centre with the broadphase's pitch and cell key (so the keys
// clamp the same way outside the measured extent), and a segment visits every cell within one cell of a cell it passes
// through.  A grid body's AABB spans at most one pitch per axis, so every point of it lies within one cell of its centre's
// cell; bodies that do not (large bodies, planes, bodies added since the last classification) are tested brute force.
// Nothing here writes anything a step reads.

struct RayIndex {
    unsigned long long *key, *key_s;     // per body: cell key (EMPTY_KEY = not in the grid), sorted
    uint32_t *body, *body_s;
    unsigned long long *hkey; uint32_t *hval; uint32_t hsize;   // cell key -> first sorted index
    uint32_t *extra;                     // [0] count, [1 ..] the bodies outside the grid (k_ray_classify)
    int *bounds;                         // 6: order-preserving min / max over the grid bodies' AABBs
};
constexpr uint32_t RAY_MISS = 0xFFFFFFFFu;   // B2D_RAY_MISS

__global__ void k_ray_reset(RayIndex x) {
    if (blockIdx.x == 0 && threadIdx.x < 6) x.bounds[threadIdx.x] = threadIdx.x < 3 ? f2ord(INFINITY) : f2ord(-INFINITY);
    if (blockIdx.x == 0 && threadIdx.x == 6) x.extra[0] = 0;
}
// After k_bp_cells: the brute-force list holds the broadphase's large bodies (F_LARGE, planes included) and every body
// whose AABB is wider than the pitch on some axis (the classification runs before a step; bodies may have been added or
// patched since).  The grid bodies' AABBs bound the walk.
__global__ void k_ray_classify(Dev d, RayIndex x) {
    float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
    GRID_STRIDE(i, d.nbodies) {
        const uint32_t f = d.flags[i];
        if (shape_of(f) == SH_NONE) continue;
        const float4 a = d.bbmin[i], b = d.bbmax[i];
        if ((f & F_LARGE) || !(b.x - a.x <= d.cell && b.y - a.y <= d.cell && b.z - a.z <= d.cell)) {
            x.key[i] = EMPTY_KEY;
            x.extra[1 + atomicAdd(&x.extra[0], 1u)] = i;
            continue;
        }
        mn[0] = fminf(mn[0], a.x); mn[1] = fminf(mn[1], a.y); mn[2] = fminf(mn[2], a.z);
        mx[0] = fmaxf(mx[0], b.x); mx[1] = fmaxf(mx[1], b.y); mx[2] = fmaxf(mx[2], b.z);
    }
    #pragma unroll
    for (int k = 0; k < 3; ++k) {
        for (int o = 16; o > 0; o >>= 1) { mn[k] = fminf(mn[k], __shfl_xor_sync(0xffffffffu, mn[k], o)); mx[k] = fmaxf(mx[k], __shfl_xor_sync(0xffffffffu, mx[k], o)); }
        if ((threadIdx.x & 31) == 0 && mn[k] <= mx[k]) { atomicMin(&x.bounds[k], f2ord(mn[k])); atomicMax(&x.bounds[3 + k], f2ord(mx[k])); }
    }
}
__global__ void k_ray_cell_starts(Dev d, RayIndex x) {
    GRID_STRIDE(i, d.nbodies) {
        const unsigned long long k = x.key_s[i];
        if (k != EMPTY_KEY && (i == 0 || x.key_s[i - 1] != k)) hash_insert(x.hkey, x.hval, x.hsize, k, i);
    }
}

struct RayBest { float f; uint32_t id, feature; v3 n; };
struct RayQuery { v3 p0, p1; uint32_t ignore1; const uint32_t *ignore; uint32_t nignore; };

B2D_D bool ray_ignored(const RayQuery &q, uint32_t j) {
    if (j == q.ignore1) return true;
    uint32_t lo = 0, hi = q.nignore;                // sorted shared list
    while (lo < hi) { const uint32_t m = (lo + hi) >> 1; if (q.ignore[m] < j) lo = m + 1; else hi = m; }
    return lo < q.nignore && q.ignore[lo] == j;
}
// One candidate.  No AABB cull in front of shape_raycast: on long segments the reference's arithmetic (the sphere
// quadratic above all) can report a hit some way off the shape, and the brute force would report it too.
B2D_D void ray_test(const Dev &d, const RayQuery &q, uint32_t j, RayBest &b) {
    const uint32_t f = d.flags[j];
    const int kind = shape_of(f);
    if (kind == SH_NONE || ray_ignored(q, j)) return;
    const RayHit h = shape_raycast(kind, d.shp[j], mk3(d.pos[j]), mkq(d.orn[j]), q.p0, q.p1);
    if (!h.hit || !(h.fraction >= 0.0f && h.fraction <= 1.0f)) return;
    if (h.fraction < b.f || (h.fraction == b.f && j < b.id)) { b.f = h.fraction; b.id = j; b.feature = h.feature; b.n = h.normal; }
}
B2D_D void ray_probe(const Dev &d, const RayIndex &x, const RayQuery &q, int cx, int cy, int cz, RayBest &b) {
    const unsigned long long key = cell_key_of(d, cx, cy, cz);
    uint32_t start;
    if (!hash_find(x.hkey, x.hval, x.hsize, key, start)) return;
    for (uint32_t k = start; k < d.nbodies && x.key_s[k] == key; ++k) ray_test(d, q, x.body_s[k], b);
}
B2D_D int ray_cell(float v, float inv_cell) { return (int)floorf(fminf(fmaxf(v * inv_cell, -1e9f), 1e9f)); }
B2D_D bool finite3(v3 v) { return fabsf(v.x) <= FLT_MAX && fabsf(v.y) <= FLT_MAX && fabsf(v.z) <= FLT_MAX; }

// The grid part of one query: clip the segment to the grid bodies' bounds (inflated by half a pitch), then a 3-D DDA
// (Amanatides & Woo) over the cells it passes.  The first cell probes its 27-cell neighbourhood; a step along axis a
// adds the 9 cells of the new far layer.  The walk stops once the best fraction lies before the current cell's exit: a
// body not probed yet has its centre more than one cell from every cell visited, so its surface is at least half a
// pitch beyond them.
B2D_D void ray_walk(const Dev &d, const RayIndex &x, const RayQuery &q, RayBest &b) {
    v3 lo = mk3(ord2f(x.bounds[0]), ord2f(x.bounds[1]), ord2f(x.bounds[2]));
    v3 hi = mk3(ord2f(x.bounds[3]), ord2f(x.bounds[4]), ord2f(x.bounds[5]));
    if (!(lo.x <= hi.x && lo.y <= hi.y && lo.z <= hi.z)) return;      // no grid bodies
    const float pad = 0.5f * d.cell;
    lo = lo - mk3(pad, pad, pad); hi = hi + mk3(pad, pad, pad);
    const v3 dir = q.p1 - q.p0;
    float ta = 0.0f, tb = 1.0f;
    #pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float o = get(q.p0, a), dd = get(dir, a), l = get(lo, a), h = get(hi, a);
        if (dd == 0.0f) { if (o < l || o > h) return; continue; }
        float t0 = (l - o) / dd, t1 = (h - o) / dd;
        if (t0 > t1) { const float s = t0; t0 = t1; t1 = s; }
        ta = fmaxf(ta, t0); tb = fminf(tb, t1);
    }
    if (!(ta <= tb)) return;
    const v3 s = q.p0 + dir * ta, e = q.p0 + dir * tb;
    // the parameter where the segment leaves cell c along axis a, from the cell index every time (an incremental
    // t += cell / |dir| drifts by a good fraction of a cell over thousands of cells)
    auto exit_t = [&](int a, int ca, int sa) { return ((float)(ca + (sa > 0 ? 1 : 0)) * d.cell - get(q.p0, a)) / get(dir, a); };
    int c[3], step[3], left[3]; float tnext[3];
    #pragma unroll
    for (int a = 0; a < 3; ++a) {
        c[a] = ray_cell(get(s, a), d.inv_cell);
        const int ce = ray_cell(get(e, a), d.inv_cell);
        step[a] = ce > c[a] ? 1 : (ce < c[a] ? -1 : 0);
        left[a] = ce > c[a] ? ce - c[a] : c[a] - ce;
        tnext[a] = step[a] ? exit_t(a, c[a], step[a]) : INFINITY;
    }
    for (int i = -1; i <= 1; ++i) for (int j = -1; j <= 1; ++j) for (int k = -1; k <= 1; ++k) ray_probe(d, x, q, c[0] + i, c[1] + j, c[2] + k, b);
    for (;;) {
        int a = -1; float t = INFINITY;
        #pragma unroll
        for (int k = 0; k < 3; ++k) if (left[k] > 0 && (a < 0 || tnext[k] < t)) { a = k; t = tnext[k]; }
        if (a < 0 || b.f < t) return;
        c[a] += step[a]; --left[a]; tnext[a] = exit_t(a, c[a], step[a]);
        const int u = (a + 1) % 3, v = (a + 2) % 3;
        int p[3]; p[a] = c[a] + step[a];
        for (int i = -1; i <= 1; ++i) for (int j = -1; j <= 1; ++j) {
            p[u] = c[u] + i; p[v] = c[v] + j;
            ray_probe(d, x, q, p[0], p[1], p[2], b);
        }
    }
}

// One thread per segment.  Zero-length and non-finite segments hit nothing.  Any output may be NULL.
__global__ void k_ray_cast(Dev d, RayIndex x, uint32_t n, const float *p0, const float *p1, const uint32_t *ignore_body,
                           const uint32_t *ignore, uint32_t nignore, uint32_t *out_body, float *out_fraction, float *out_normal,
                           uint32_t *out_feature) {
    GRID_STRIDE(r, n) {
        RayQuery q;
        q.p0 = mk3(p0[3 * r], p0[3 * r + 1], p0[3 * r + 2]); q.p1 = mk3(p1[3 * r], p1[3 * r + 1], p1[3 * r + 2]);
        q.ignore1 = ignore_body ? ignore_body[r] : RAY_MISS; q.ignore = ignore; q.nignore = nignore;
        RayBest b; b.f = SCALAR_MAX; b.id = RAY_MISS; b.feature = RAY_FEATURE_NONE; b.n = mk3(0, 0, 0);
        const bool degenerate = q.p0.x == q.p1.x && q.p0.y == q.p1.y && q.p0.z == q.p1.z;
        if (!degenerate && finite3(q.p0) && finite3(q.p1)) {
            const uint32_t ne = x.extra[0];
            for (uint32_t k = 0; k < ne; ++k) ray_test(d, q, x.extra[1 + k], b);
            ray_walk(d, x, q, b);
        }
        if (out_body) out_body[r] = b.id;
        if (out_fraction) out_fraction[r] = b.f;
        if (out_normal) { out_normal[3 * r] = b.n.x; out_normal[3 * r + 1] = b.n.y; out_normal[3 * r + 2] = b.n.z; }
        if (out_feature) out_feature[r] = b.feature;
    }
}

} // namespace b2d
