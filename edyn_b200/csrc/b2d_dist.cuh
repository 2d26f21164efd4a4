// Multi-GPU side of the hot path (SURVEY.md section 8e, DESIGN.md section 5): islands are the unit of distribution, one
// world per GPU.  Everything a rank has to tell its peers is produced on the device, straight into buffers the host
// framework hands to NCCL:
//   * the box of the rank's dynamic bodies (k_bounds_*, b2d_kernels.cuh), every step;
//   * when two rank boxes come within the broadphase margin: the AABBs of the islands near the peer
//     (update_island_aabbs, /root/reference/src/edyn/sys/update_aabbs.cpp:106-138) -> k_ibox_*, k_halo_collect;
//   * the hand-over plan: an island that touches an island of a lower rank moves there, whole
//     (merge_islands "move into the other island", src/edyn/simulation/island_manager.cpp:297-350) -> k_plan_*;
//   * the hand-over blob: bodies with their current state, the manifolds (points, lifetimes, warm-start impulses),
//     joints and collision exclusions attached to them, named by scene-global entity -> k_pack_*, k_unpack_*.
// Also here: dirty-subset staging of body components (k_patch_bodies; SURVEY section 8b,
// include/edyn/comp/shared_comp.hpp:36-86 is the component list the reference replicates the same way).
#pragma once
#include "b2d_kernels.cuh"

namespace b2d {

constexpr uint32_t NO_RANK = 0xFFFFFFFFu;
constexpr float HALO_MARGIN = BREAKING_THRESHOLD * 1.3f;      // manifold separation threshold, broadphase.hpp:18

// ---------------------------------------------------------------- entity names

B2D_D void ehash_insert(unsigned long long *tab, uint32_t size, uint32_t entity, uint32_t local) {
    uint32_t h = hash64(entity) & (size - 1);
    const unsigned long long v = ((unsigned long long)entity << 32) | local;
    for (;;) {
        unsigned long long prev = atomicCAS(&tab[h], EMPTY_KEY, v);
        if (prev == EMPTY_KEY) return;
        if ((uint32_t)(prev >> 32) == entity) { tab[h] = v; return; }      // re-named: latest wins
        h = (h + 1) & (size - 1);
    }
}
B2D_D uint32_t ehash_find(const unsigned long long *tab, uint32_t size, uint32_t entity) {
    uint32_t h = hash64(entity) & (size - 1);
    for (;;) {
        unsigned long long cur = tab[h];
        if (cur == EMPTY_KEY) return 0xFFFFFFFFu;
        if ((uint32_t)(cur >> 32) == entity) return (uint32_t)cur;
        h = (h + 1) & (size - 1);
    }
}
__global__ void k_entities_default(Dev d, uint32_t first, uint32_t n) {
    GRID_STRIDE(k, n) { d.entity[first + k] = first + k; }
}
__global__ void k_entities_set(Dev d, uint32_t first, uint32_t n, const uint32_t *ent) {
    GRID_STRIDE(k, n) { d.entity[first + k] = ent[k]; }
}
// the table is rebuilt from the entity array (names may have been reassigned)
__global__ void k_ehash_build(Dev d) {
    GRID_STRIDE(i, d.nbodies) { if (!(d.flags[i] & F_REMOVED)) ehash_insert(d.ehash, d.ehash_size, d.entity[i], i); }
}

// ---------------------------------------------------------------- broadphase classes
// F_LARGE (brute-force list instead of the grid) is re-derived by the host whenever the body population changes
__global__ void k_large_clear(Dev d) { GRID_STRIDE(i, d.nbodies) d.flags[i] &= ~F_LARGE; }
__global__ void k_large_set(Dev d) { GRID_STRIDE(k, d.nlarge) d.flags[d.large_list[k]] |= F_LARGE; }

// ---------------------------------------------------------------- dirty-subset staging

struct Patch {      // device copies of the host arrays, nullptr = component untouched
    const float *pos, *orn, *linvel, *angvel, *inv_mass, *inv_inertia, *gravity, *friction, *restitution;
    const uint32_t *kind;
    const uint32_t *material;       // material ids; the host has refused changes between sensor and non-sensor
};
// registry.patch / replace on a subset of bodies: only the named components change; AABB and inertia_world_inv follow
// the transform the way solver.cpp:453-465 refreshes them.  A kind change re-derives what make_rigidbody sets per kind
// (util/rigidbody.cpp:62-118): non-dynamic bodies have no mass, static ones no velocity.
__global__ void k_patch_bodies(Dev d, const uint32_t *ids, uint32_t n, Patch p) {
    GRID_STRIDE(k, n) {
        const uint32_t i = ids[k];
        uint32_t f = d.flags[i];
        if (f & F_REMOVED) continue;
        if (p.kind) f = (f & ~F_KIND_MASK) | (p.kind[k] & F_KIND_MASK);
        const bool dyn = (f & F_KIND_MASK) == 0u;
        float4 p4 = d.pos[i];
        if (p.pos) { p4.x = p.pos[3 * k]; p4.y = p.pos[3 * k + 1]; p4.z = p.pos[3 * k + 2]; }
        if (p.inv_mass) p4.w = p.inv_mass[k];
        if (!dyn) p4.w = 0.0f;
        d.pos[i] = p4;
        if (p.orn) d.orn[i] = make_float4(p.orn[4 * k], p.orn[4 * k + 1], p.orn[4 * k + 2], p.orn[4 * k + 3]);
        if ((f & F_KIND_MASK) == 2u) { d.linvel[i] = make_float4(0, 0, 0, 0); d.angvel[i] = make_float4(0, 0, 0, 0); }
        else {
            if (p.linvel) d.linvel[i] = make_float4(p.linvel[3 * k], p.linvel[3 * k + 1], p.linvel[3 * k + 2], 0);
            if (p.angvel) d.angvel[i] = make_float4(p.angvel[3 * k], p.angvel[3 * k + 1], p.angvel[3 * k + 2], 0);
        }
        if (p.inv_inertia) for (int r = 0; r < 3; ++r) d.invI[3 * (size_t)i + r] = make_float4(p.inv_inertia[9 * k + 3 * r], p.inv_inertia[9 * k + 3 * r + 1], p.inv_inertia[9 * k + 3 * r + 2], 0);
        if (!dyn) for (int r = 0; r < 3; ++r) d.invI[3 * (size_t)i + r] = make_float4(0, 0, 0, 0);
        if (p.gravity) d.grav[i] = make_float4(p.gravity[3 * k], p.gravity[3 * k + 1], p.gravity[3 * k + 2], 0);
        float2 m = d.mat[i];
        if (p.friction) m.x = p.friction[k];
        if (p.restitution) m.y = p.restitution[k];
        d.mat[i] = m;
        if (p.material && !(f & F_SENSOR)) d.matid[i] = p.material[k];
        f &= ~F_SLEEPING;                       // a patched body is awake (registry.patch wakes the island)
        d.flags[i] = f;
        const v3 pos = mk3(d.pos[i]); const q4 orn = mkq(d.orn[i]);
        if (is_dynamic(f)) store_invIW(d, i, world_inertia(orn, load_m3(d.invI, i)), p4.w);
        else store_invIW(d, i, m3_zero(), 0.0f);
        const int sk = shape_of(f);
        if (sk != SH_NONE) { box3 bb = shape_aabb(sk, d.shp[i], pos, orn); d.bbmin[i] = f4(bb.mn, 0); d.bbmax[i] = f4(bb.mx, 0); }
    }
}

// ---------------------------------------------------------------- island AABBs near a peer

__global__ void k_ibox_init(Dev d) {
    GRID_STRIDE(i, d.nbodies) {
        int *b = d.ibox + 6 * (size_t)i;
        b[0] = b[1] = b[2] = f2ord(INFINITY); b[3] = b[4] = b[5] = f2ord(-INFINITY);
        d.isl_dst[i] = NO_RANK;
    }
}
// update_island_aabbs (sys/update_aabbs.cpp:106-138): union over the procedural members, kept at the island's root
__global__ void k_ibox_reduce(Dev d) {
    GRID_STRIDE(i, d.nbodies) {
        const uint32_t f = d.flags[i];
        if (!is_procedural(f) || shape_of(f) == SH_NONE) continue;
        const uint32_t r = d.parent[i];
        if (r == 0xFFFFFFFFu) continue;
        int *b = d.ibox + 6 * (size_t)r;
        const float4 a = d.bbmin[i], c = d.bbmax[i];
        atomicMin(&b[0], f2ord(a.x)); atomicMin(&b[1], f2ord(a.y)); atomicMin(&b[2], f2ord(a.z));
        atomicMax(&b[3], f2ord(c.x)); atomicMax(&b[4], f2ord(c.y)); atomicMax(&b[5], f2ord(c.z));
    }
}
struct HaloRec { float mn[3], mx[3]; uint32_t label, rank; };      // 32 B on the wire
B2D_D bool boxes_touch(const float *amn, const float *amx, const float *bmn, const float *bmx, float margin) {
    return amn[0] - margin <= bmx[0] && amx[0] + margin >= bmn[0] && amn[1] - margin <= bmx[1] && amx[1] + margin >= bmn[1] &&
           amn[2] - margin <= bmx[2] && amx[2] + margin >= bmn[2];
}
// islands whose AABB, inflated by the margin, reaches into the box of one of the peers in `peer_mask`
__global__ void k_halo_collect(Dev d, const float *boxes, uint32_t nboxes, uint32_t self, unsigned long long peer_mask,
                               HaloRec *out, uint32_t capacity, uint32_t *count) {
    GRID_STRIDE(i, d.nbodies) {
        if (!is_procedural(d.flags[i]) || d.parent[i] != i) continue;
        const int *b = d.ibox + 6 * (size_t)i;
        HaloRec r;
        for (int k = 0; k < 3; ++k) { r.mn[k] = ord2f(b[k]); r.mx[k] = ord2f(b[3 + k]); }
        if (!(r.mn[0] <= r.mx[0])) continue;                         // no shaped member
        bool hit = false;
        for (uint32_t p = 0; p < nboxes && !hit; ++p) {
            if (p == self || !((peer_mask >> p) & 1ULL)) continue;
            hit = boxes_touch(r.mn, r.mx, boxes + 6 * p, boxes + 6 * p + 3, d.halo_margin);
        }
        if (!hit) continue;
        const uint32_t k = atomicAdd(count, 1u);
        if (k < capacity) { r.label = i; r.rank = self; out[k] = r; }
    }
}

// ---------------------------------------------------------------- hand-over plan

// recs: the halo records of all ranks, concatenated in rank order; [my_b, my_e) are this rank's, [0, my_b) belong to
// lower ranks.  An island of mine that touches an island of a lower rank goes to the lowest such rank.
__global__ void k_plan_islands(Dev d, const HaloRec *recs, uint32_t my_b, uint32_t my_e) {
    const unsigned long long total = (unsigned long long)(my_e - my_b) * my_b;
    for (unsigned long long t = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; t < total; t += (unsigned long long)gridDim.x * blockDim.x) {
        const uint32_t i = my_b + (uint32_t)(t / my_b), j = (uint32_t)(t % my_b);
        const HaloRec a = recs[i], b = recs[j];
        if (boxes_touch(a.mn, a.mx, b.mn, b.mx, d.halo_margin)) atomicMin(&d.isl_dst[a.label], b.rank);
    }
}
// counts: per destination rank {bodies, manifolds, hinges, 0}
__global__ void k_plan_bodies(Dev d, uint32_t *counts) {
    GRID_STRIDE(i, d.nbodies) {
        uint32_t dst = NO_RANK;
        if (is_procedural(d.flags[i])) { const uint32_t r = d.parent[i]; if (r != 0xFFFFFFFFu) dst = d.isl_dst[r]; }
        d.bdst[i] = dst;
        if (dst != NO_RANK) atomicAdd(&counts[4 * dst], 1u);
    }
}
B2D_D uint32_t pair_dst(const Dev &d, uint2 p) { const uint32_t a = d.bdst[p.x]; return a != NO_RANK ? a : d.bdst[p.y]; }
__global__ void k_plan_constraints(Dev d, uint32_t *counts) {
    const uint32_t hwm = d.cnt->hwm;
    GRID_STRIDE(m, hwm + d.nhinges) {
        uint2 p;
        if (m < hwm) { if (!(d.mstate[m] & MS_ALIVE)) continue; p = d.mpair[m]; }
        else p = d.hpair[m - hwm];
        const uint32_t dst = pair_dst(d, p);
        if (dst != NO_RANK) atomicAdd(&counts[4 * dst + (m < hwm ? 1 : 2)], 1u);
    }
}

// ---------------------------------------------------------------- hand-over blob
// header (4 x uint4) | bodies: 13 float4 each | manifolds: 21 float4 each | hinges: 7 float4 each | exclusions: uint2 each
// A body's flags carry F_SENSOR and F_PRESENT; its material id sits in o[10].z, its present transform in o[11], o[12].
constexpr uint32_t BLOB_MAGIC = 0xB2D0B10Bu;
constexpr uint32_t BLOB_BODY_F4 = 13, BLOB_MANIFOLD_F4 = 21, BLOB_HINGE_F4 = 7;
struct BlobHeader { uint32_t magic, nb, nm, nh, nx; uint32_t pad[11]; };      // 64 B
static_assert(sizeof(BlobHeader) == 64, "blob header is four 16-byte words");
B2D_D float fbits(uint32_t u) { return __uint_as_float(u); }
B2D_D uint32_t ubits(float f) { return __float_as_uint(f); }

__global__ void k_pack_header(BlobHeader *h, uint32_t nb, uint32_t nm, uint32_t nh, uint32_t nx) {
    if (blockIdx.x == 0 && threadIdx.x == 0) { h->magic = BLOB_MAGIC; h->nb = nb; h->nm = nm; h->nh = nh; h->nx = nx; }
}
__global__ void k_pack_bodies(Dev d, const uint32_t *ids, uint32_t n, float4 *out) {
    GRID_STRIDE(k, n) {
        const uint32_t i = ids[k];
        float4 *o = out + (size_t)BLOB_BODY_F4 * k;
        const uint32_t f = d.flags[i];
        const float4 lv = d.linvel[i], av = d.angvel[i], g = d.grav[i];
        const float2 m = d.mat[i];
        const unsigned long long grp = d.group[i], msk = d.fmask[i];
        o[0] = d.pos[i]; o[1] = d.orn[i];
        o[2] = make_float4(lv.x, lv.y, lv.z, fbits(f & ~F_SLEEPING));
        o[3] = make_float4(av.x, av.y, av.z, fbits(d.entity[i]));
        o[4] = d.invI[3 * (size_t)i]; o[5] = d.invI[3 * (size_t)i + 1]; o[6] = d.invI[3 * (size_t)i + 2];
        o[7] = g; o[8] = d.shp[i];
        o[9] = make_float4(m.x, m.y, fbits((uint32_t)grp), fbits((uint32_t)(grp >> 32)));
        o[10] = make_float4(fbits((uint32_t)msk), fbits((uint32_t)(msk >> 32)), fbits(d.matid[i]), 0);
        o[11] = d.ppos[i]; o[12] = d.porn[i];
    }
}
// flags for the deterministic compaction (slot order) of the constraints that leave for `dst`
__global__ void k_pack_flag_manifolds(Dev d, uint32_t dst) {
    const uint32_t hwm = d.cnt->hwm;
    GRID_STRIDE(m, d.NM) {
        uint32_t fl = 0;
        if (m < hwm && (d.mstate[m] & MS_ALIVE) && pair_dst(d, d.mpair[m]) == dst) fl = 1;
        d.free_flag[m] = fl;
    }
}
__global__ void k_pack_manifolds(Dev d, float4 *out) {
    const uint32_t hwm = d.cnt->hwm;
    GRID_STRIDE(m, hwm) {
        if (!d.free_flag[m]) continue;
        float4 *o = out + (size_t)BLOB_MANIFOLD_F4 * d.free_rank[m];
        const uint2 p = d.mpair[m];
        const uint32_t np = d.mstate[m] & MS_NPTS_MASK;
        o[0] = make_float4(fbits(d.entity[p.x]), fbits(d.entity[p.y]), fbits(np), 0);
        for (uint32_t s = 0; s < 4; ++s) {
            const size_t i = (size_t)s * d.NM + m;
            const bool on = s < np;
            const float4 z = make_float4(0, 0, 0, 0);
            o[1 + 5 * s] = on ? d.pA[i] : z; o[2 + 5 * s] = on ? d.pB[i] : z; o[3 + 5 * s] = on ? d.pN[i] : z;
            o[4 + 5 * s] = on ? d.pL[i] : z; o[5 + 5 * s] = on ? d.pI[i] : z;
        }
    }
}
__global__ void k_pack_flag_hinges(Dev d, uint32_t dst) {
    GRID_STRIDE(h, d.NH) {
        uint32_t fl = 0;
        if (h < d.nhinges) { const uint2 p = d.hpair[h]; if (p.x != p.y && pair_dst(d, p) == dst) fl = 1; }
        d.hidx[h] = fl;
    }
}
__global__ void k_pack_hinges(Dev d, float4 *out) {
    GRID_STRIDE(h, d.nhinges) {
        if (!d.hidx[h]) continue;
        float4 *o = out + (size_t)BLOB_HINGE_F4 * d.hidx_s[h];
        const uint2 p = d.hpair[h];
        const float *imp = d.himp + 5 * (size_t)h;
        const float4 pa = d.hpivA[h], pb = d.hpivB[h], f0 = d.hfA0[h];
        o[0] = make_float4(fbits(d.entity[p.x]), fbits(d.entity[p.y]), imp[0], imp[1]);
        o[1] = make_float4(pa.x, pa.y, pa.z, imp[2]); o[2] = make_float4(pb.x, pb.y, pb.z, imp[3]);
        o[3] = make_float4(f0.x, f0.y, f0.z, imp[4]); o[4] = d.hfA1[h]; o[5] = d.hfA2[h]; o[6] = d.hfB0[h];
    }
}
// exclusion pairs arrive in local ids (host list), leave as entities
__global__ void k_pack_exclusions(Dev d, const uint2 *local, uint32_t n, uint2 *out) {
    GRID_STRIDE(k, n) { out[k] = make_uint2(d.entity[local[k].x], d.entity[local[k].y]); }
}

// (F_LARGE is a property of the receiving world's grid: the host re-classifies before the next step)
__global__ void k_unpack_bodies(Dev d, uint32_t first, uint32_t n, const float4 *in) {
    GRID_STRIDE(k, n) {
        const uint32_t i = first + k;
        const float4 *o = in + (size_t)BLOB_BODY_F4 * k;
        const uint32_t f = ubits(o[2].w) & ~(F_LARGE | F_SLEEPING | F_REMOVED);
        d.pos[i] = o[0]; d.orn[i] = o[1];
        d.linvel[i] = make_float4(o[2].x, o[2].y, o[2].z, 0); d.angvel[i] = make_float4(o[3].x, o[3].y, o[3].z, 0);
        d.entity[i] = ubits(o[3].w);
        d.invI[3 * (size_t)i] = o[4]; d.invI[3 * (size_t)i + 1] = o[5]; d.invI[3 * (size_t)i + 2] = o[6];
        d.grav[i] = o[7]; d.shp[i] = o[8];
        d.mat[i] = make_float2(o[9].x, o[9].y);
        d.group[i] = (unsigned long long)ubits(o[9].z) | ((unsigned long long)ubits(o[9].w) << 32);
        d.fmask[i] = (unsigned long long)ubits(o[10].x) | ((unsigned long long)ubits(o[10].y) << 32);
        d.matid[i] = ubits(o[10].z);
        d.ppos[i] = o[11]; d.porn[i] = o[12];
        d.flags[i] = f;
        ehash_insert(d.ehash, d.ehash_size, d.entity[i], i);
    }
}
// new manifolds go behind the high-water mark in blob order (the sender's slot order)
__global__ void k_unpack_manifolds(Dev d, uint32_t n, const float4 *in, uint32_t base) {
    GRID_STRIDE(k, n) {
        const float4 *o = in + (size_t)BLOB_MANIFOLD_F4 * k;
        const uint32_t m = base + k;
        const uint32_t a = ehash_find(d.ehash, d.ehash_size, ubits(o[0].x)), b = ehash_find(d.ehash, d.ehash_size, ubits(o[0].y));
        if (a == 0xFFFFFFFFu || b == 0xFFFFFFFFu) { atomicOr(&d.cnt->err, ERR_UNKNOWN_ENTITY); d.mstate[m] = COLOR_NONE << MS_COLOR_SHIFT; continue; }
        const uint32_t np = ubits(o[0].z) & MS_NPTS_MASK;
        d.mpair[m] = make_uint2(a, b);
        d.mstate[m] = MS_ALIVE | (COLOR_NONE << MS_COLOR_SHIFT) | np;
        for (uint32_t s = 0; s < 4; ++s) {
            const size_t i = (size_t)s * d.NM + m;
            d.pA[i] = o[1 + 5 * s]; d.pB[i] = o[2 + 5 * s]; d.pN[i] = o[3 + 5 * s]; d.pL[i] = o[4 + 5 * s]; d.pI[i] = o[5 + 5 * s];
        }
    }
}
__global__ void k_unpack_hinges(Dev d, uint32_t first, uint32_t n, const float4 *in) {
    GRID_STRIDE(k, n) {
        const float4 *o = in + (size_t)BLOB_HINGE_F4 * k;
        const uint32_t h = first + k;
        uint32_t a = ehash_find(d.ehash, d.ehash_size, ubits(o[0].x)), b = ehash_find(d.ehash, d.ehash_size, ubits(o[0].y));
        if (a == 0xFFFFFFFFu || b == 0xFFFFFFFFu) { atomicOr(&d.cnt->err, ERR_UNKNOWN_ENTITY); a = b = 0; }      // parked like a removed joint
        d.hpair[h] = make_uint2(a, b);
        d.hpivA[h] = make_float4(o[1].x, o[1].y, o[1].z, 0); d.hpivB[h] = make_float4(o[2].x, o[2].y, o[2].z, 0);
        d.hfA0[h] = make_float4(o[3].x, o[3].y, o[3].z, 0); d.hfA1[h] = o[4]; d.hfA2[h] = o[5]; d.hfB0[h] = o[6];
        float *imp = d.himp + 5 * (size_t)h;
        imp[0] = o[0].z; imp[1] = o[0].w; imp[2] = o[1].w; imp[3] = o[2].w; imp[4] = o[3].w;
        d.hcolor[h] = COLOR_NONE;
    }
}
__global__ void k_unpack_exclusions(Dev d, const uint2 *ent, uint32_t n, uint2 *local) {
    GRID_STRIDE(k, n) { local[k] = make_uint2(ehash_find(d.ehash, d.ehash_size, ent[k].x), ehash_find(d.ehash, d.ehash_size, ent[k].y)); }
}
// collision_exclusion pairs appended to the device table (keys are known not to be in it)
__global__ void k_xhash_insert(Dev d, const unsigned long long *keys, uint32_t n) {
    GRID_STRIDE(k, n) hash_insert(d.xhash_key, nullptr, d.xhash_size, keys[k], 0u);
}
__global__ void k_bump_hwm(Dev d, uint32_t n) {
    if (blockIdx.x == 0 && threadIdx.x == 0) d.cnt->hwm = min(d.NM, d.cnt->hwm + n);
}

} // namespace b2d
