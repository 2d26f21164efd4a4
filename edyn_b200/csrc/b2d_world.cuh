// Device-resident world: SoA layout in HBM (DESIGN.md section 3).  All per-body and per-contact arrays are
// float4 so every access is one 16 B vector load; manifold point arrays are slot-major
// (index = slot * max_manifolds + manifold) so a warp reading slot s of 32 consecutive manifolds
// touches 512 contiguous bytes.
#pragma once
#include "b2d_math.cuh"

namespace b2d {

// flags word per body
constexpr uint32_t F_KIND_MASK = 3u;          // 0 dynamic, 1 kinematic, 2 static (B2D_DYNAMIC..)
constexpr uint32_t F_SHAPE_SHIFT = 4;         // bits 4..11 shape kind
constexpr uint32_t F_ROLLING = 1u << 12;      // rolling_tag (util/rigidbody.cpp:120-130)
constexpr uint32_t F_SENSOR = 1u << 17;       // no material component: its manifolds get points but no rows (collision_util.cpp:358-384)
constexpr uint32_t F_FILTER = 1u << 13;       // has collision_filter
constexpr uint32_t F_LARGE = 1u << 14;        // larger than a broadphase cell: brute-force list
constexpr uint32_t F_SLEEPING = 1u << 16;     // sleeping_tag: excluded from every per-step view until its island wakes
constexpr uint32_t F_REMOVED = 1u << 15;      // destroyed (b2d_remove_bodies): static, shapeless, its manifolds and joints die
constexpr uint32_t F_PRESENT = 1u << 18;      // has present_position + present_orientation (k_presentation only; no step kernel reads it)

constexpr uint32_t MATERIAL_UNASSIGNED = 0xFFFFu;   // material::UnassignedID: never in the mixing table

// mstate word per manifold slot
constexpr uint32_t MS_NPTS_MASK = 7u;
constexpr uint32_t MS_ALIVE = 1u << 7;
constexpr uint32_t MS_COLOR_SHIFT = 8;        // bits 8..15 colour, 0xFF = none
constexpr uint32_t MS_COLOR_MASK = 0xFFu << MS_COLOR_SHIFT;
constexpr uint32_t COLOR_NONE = 0xFFu;
constexpr int MAX_COLORS = 64;
// Island tiles (DESIGN.md section 2): islands small enough to be solved inside one CTA -- body records in shared memory,
// constraint rows in registers for all iterations, __syncthreads between colours, no global synchronisation at all --
// are packed into tiles of up to TILE_CAP bodies / contact manifolds / joints; everything else (a pile is one island)
// goes through the global dataflow kernels.
#ifndef B2D_TILE_CAP
#define B2D_TILE_CAP 256
#endif
constexpr int TILE_CAP = B2D_TILE_CAP;         // threads per tile CTA = capacity in bodies, manifolds and joints
constexpr int TILE_ISLAND_MAX = TILE_CAP / 2;  // an island is tiled if it has at most this many bodies, manifolds and joints
constexpr uint32_t TILE_NONE = 0xFFFFFFFFu;
constexpr uint32_t ISL_MULTIPOINT = 0x80000000u;  // isl_nm flag: a manifold of the island has more than 2 points
constexpr uint32_t SLOT_NONE = 0xFFFFu;
// sort keys.  tiled: tile(16) | colour(6); dataflow: DF | colour(6) | points-1 (2) | spatial rank(14); no rows: INACTIVE
constexpr int KEY_TILE_BITS = 16;                                   // 24-bit keys: three radix passes
constexpr uint32_t KEY_DF = 1u << (KEY_TILE_BITS + 6);
constexpr uint32_t KEY_INACTIVE = 1u << (KEY_TILE_BITS + 7);
constexpr int COLOR_KEY_BITS = KEY_TILE_BITS + 8;
constexpr int KEY_DF_SPATIAL_BITS = 14;
constexpr int KEY_DF_COLOR_SHIFT = KEY_DF_SPATIAL_BITS + 2;
// broadphase: cells of the direct cell table per body (Dev::cstart); an occupied box with more cells uses the cell hash
constexpr uint32_t DENSE_CELLS_PER_BODY = 4;

constexpr uint32_t ERR_MANIFOLD_CAPACITY = 1u;
constexpr uint32_t ERR_COLOR_OVERFLOW = 2u;
constexpr uint32_t ERR_LARGE_CAPACITY = 4u;
constexpr uint32_t ERR_UNKNOWN_ENTITY = 16u;    // a hand-over blob names a body this world does not hold
constexpr uint32_t ERR_RESTITUTION_GROUP = 32u; // restitution solver: one body touches more manifolds / points than a group holds
constexpr uint32_t ERR_SOLVER_TIMEOUT = 8u;     // a dataflow wait exceeded its spin budget (would have been a hang)

struct Counters {
    uint32_t hwm;            // manifold slots in use are [0, hwm)
    uint32_t nfree;          // dead slots below hwm this step
    uint32_t nnew;           // pairs found this step
    uint32_t nactive;        // manifolds with >= 1 point, i.e. rows in the solver arrays
    uint32_t ncolors;        // contact colours in use
    uint32_t nhcolors;       // hinge colours in use
    uint32_t err;
    uint32_t remaining[2];   // colouring loop: uncoloured constraints, double buffered per round
    uint32_t npoints;        // contact points (statistics)
    uint32_t nislands;
    uint32_t nlist;          // colouring work list length
    uint32_t bar;            // grid barrier counter (zeroed by the host before each persistent kernel)
    int bounds[6];           // order-preserving int encoding of the min/max of all dynamic AABBs (multi-GPU exchange)
    uint32_t speed;          // float bits: fastest point of any dynamic body, m/s (multi-GPU exchange)
    uint32_t nhactive;               // hinges with rows this step
    uint32_t ntiles;                 // island tiles this step
    uint32_t ntiles2;                // of which two-point tiles: [0, ntiles2); generic tiles [ntiles2, ntiles)
    uint32_t tile_wmax;              // heaviest tiled island (zeroed by the host, like the next two)
    uint32_t ncolors_all, nhcolors_all;      // colours in use over both solver paths (statistics)
    uint32_t ntiled, nhtiled;        // contact manifolds / hinges solved in tiles: [0, ntiled) of the sorted arrays
    uint32_t coff[MAX_COLORS + 2];   // dataflow path: start of each contact colour in the sorted arrays
    uint32_t hoff[MAX_COLORS + 2];   // same for hinges
    uint32_t cchunk[MAX_COLORS + 2]; // prefix sum of ceil(colour size / 32): warp-sized chunks never span two colours
    uint32_t hchunk[MAX_COLORS + 2];
    uint32_t npoff[16];              // narrowphase: start of each pair-type range in the type-sorted list
    uint32_t npcount[16], npcursor[16];      // its histogram and scatter cursors (zeroed by the host)
    // Island rebuild reuse.  graph_changed is set by whatever changes an input of the island rebuild (connected
    // components, colouring, tile packing, sort keys and sorts: a pure function of the constraint graph) and cleared
    // by the rebuild; a CUDA-graph step skips the rebuild while it is clear (b2d_api.cu enqueue_front).
    uint32_t graph_changed;
    unsigned long long steps_rebuilt, steps_reused;          // graph steps that ran / skipped the rebuild (statistics)
    unsigned long long dbg[16];  // development counters (B2D_DF_PROFILE builds only)
    uint32_t bp_direct;          // this step's cell lookup: 1 the direct table (Dev::cstart), 0 the cell hash (k_bp_cell_mode)
    uint32_t bp_count_walk;      // the last thread-per-body count pass: 1 the whole neighbourhood, 2 half of it (k_bp_pairs)
};

struct Dev {
    uint32_t NB, NM, NH;           // capacities
    uint32_t nbodies, nhinges, nlarge;   // host-known counts
    float dt;
    float cell, inv_cell;          // broadphase grid pitch
    float halo_margin;             // multi-GPU: islands closer than this to a peer's box / island are boundary islands
    int cell_org[3]; int cell_bits[3];     // broadphase cell key: origin and field widths (bits) per axis

    // ---- bodies
    float4 *pos;       // xyz position, w inv_mass
    float4 *orn;
    float4 *linvel, *angvel;
    float4 *dvw;       // [2*i] delta_linvel, [2*i+1] delta_angvel
    float4 *invI;      // 3 rows, body space
    float4 *invIW;     // 3 rows, world space; row0.w = inv_mass (0 unless dynamic)
    float4 *grav;
    float4 *shp;
    float4 *bbmin, *bbmax;
    uint32_t *flags;
    float2 *mat;       // friction, restitution
    unsigned long long *group, *fmask;

    // ---- broadphase scratch
    unsigned long long *cellkey, *cellkey_s;
    uint32_t *cellbody, *cellbody_s;
    uint32_t *brank;                     // position of every body in the sorted cell order (spatial rank)
    float4 *bprec_min, *bprec_max;       // per sorted index: the body's AABB min | id and max | flags (candidate records)
    uint32_t *cell_box;                  // occupied key fields this step: min x, y, z, then min of ~x, ~y, ~z (k_bp_cells)
    // ---- island tiles
    uint32_t max_tiles;
    uint32_t *isl_nb, *isl_nm, *isl_nh;  // per island root: dynamic bodies, manifolds with points (| ISL_MULTIPOINT), joints
    unsigned long long *swgt, *swsum;    // per body id: packing weight of the island it is the root of (two-point islands in
                                         // the low word, the others in the high word), exclusive prefix sum
    uint32_t *btile, *bslot;             // per body: tile of its island (TILE_NONE: dataflow path), record slot in the tile
    uint32_t *tile_nb, *tile_body;       // per tile: bodies, slot -> body (TILE_CAP per tile)
    uint32_t *tile_c0, *tile_c1, *tile_h0, *tile_h1;   // per tile: its range of the sorted contact / hinge arrays
    unsigned long long *chash_key; uint32_t *chash_val; uint32_t chash_size;
    uint32_t *cstart; uint32_t cstart_size;   // direct cell table: first sorted index per cell of the occupied box (k_bp_cell_starts)
    uint32_t *large_list;
    uint32_t *lmask;                     // per body: bit k set while an alive manifold joins it to large_list[k], k < 32 (k_bp_separate)
    uint32_t *newcount, *newoff;
    uint2 *newpairs;
    uint32_t *free_flag, *free_rank, *free_list;
    unsigned long long *mhash_key; uint32_t *mhash_val; uint32_t mhash_size;
    unsigned long long *xhash_key; uint32_t xhash_size;    // exclusion pairs (0 = none)

    // ---- manifolds (slot-major point arrays)
    uint2 *mpair;
    uint32_t *mstate;
    float4 *pA;        // pivotA xyz, distance
    float4 *pB;        // pivotB xyz, friction
    float4 *pN;        // normal xyz, restitution
    float4 *pL;        // local_normal xyz, bits(att | lifetime << 2)
    float4 *pI;        // normal impulse, friction impulse[2], unused

    // ---- islands / colouring
    uint32_t *parent;
    unsigned long long *bmask, *jmask;      // colours in use per body (contacts / hinges)
    unsigned long long *prop, *jprop;
    uint32_t *ckey, *ckey_s; uint32_t *cidx, *cidx_s;
    uint32_t *clist;             // colouring work list (manifold slots with points)
    uint32_t *hkey, *hkey_s; uint32_t *hidx, *hidx_s;
    uint32_t *isl_err; uint32_t *isl_done;

    // ---- solver rows, colour-sorted order (index = slot * NM + sorted position)
    uint4 *hdr;        // body a, body b, npts, shared-memory slots (a | b << 16); the manifold slot is cidx_s[i]
    float4 *R0;        // normal xyz, rhs_n
    float4 *R1;        // rA xyz, eff_mass_n
    float4 *R2;        // rB xyz, friction
    float4 *R3;        // eff_mass_t0, eff_mass_t1, rhs_t0, rhs_t1
    float4 *IMP;       // impulse n, t0, t1

    // ---- hinges
    uint2 *hpair;
    float4 *hpivA, *hpivB;       // pivot in body space
    float4 *hfA0, *hfA1, *hfA2;  // frame[0] columns (axis, p, q)
    float4 *hfB0;                // frame[1] column 0 (axis)
    float *himp;                 // 5 per hinge
    uint32_t *hcolor;
    float4 *HR;                  // 7 float4 per sorted hinge: rA|eff0, rB|eff1, p|eff2, q|eff3, (eff4,rhs0,rhs1,rhs2), (rhs3,rhs4,imp0,imp1), (imp2,imp3,imp4,0)
    uint4 *hhdr;                 // a, b, hinge id, shared-memory slots (a | b << 16)

    // ---- dataflow schedule of the velocity solve
    // island sleeping (island_manager.cpp:541-623); arrays are indexed by body id, island data sits at the root's id
    uint32_t sleeping;                   // enabled (B2D_FLAG_SLEEPING)
    uint32_t *prev_label, *isl_size, *size_new, *isl_flags;
    unsigned long long *contributor, *heir;
    double *isl_ts, *ts_new;
    uint32_t *pisl, *hisl;       // per sorted constraint: island label (position solver early exit)
    float4 *prec;                // position solver: 3 float4 per body, (pos,t) (orn.xyz,t) (orn.w,fresh,0,t)
    uint2 *tkt, *htkt;           // per sorted constraint, per body side: S | base << 8 | k << 16 (see ticket_word)

    // ---- multi-GPU hand-over (b2d_dist.cuh): scene-global body names and the island / destination scratch
    uint32_t *entity;                    // scene-global name per body (entt::entity in the EnTT binding); default = local id
    unsigned long long *ehash; uint32_t ehash_size;      // entity -> local id, open addressing, key << 32 | value
    int *ibox;                           // 6 ints per body id: order-preserving encoding of the island AABB, stored at the root
    uint32_t *isl_dst, *bdst;            // destination rank per island root / per body (0xFFFFFFFF = stays)

    Counters *cnt;

    // ---- restitution solver (B2D_FLAG_RESTITUTION_SOLVER; appended last so that the other fields keep their offsets)
    uint32_t rest_iters, rest_individual;    // settings.num_restitution_iterations / num_individual_restitution_iterations; 0 = off
    uint32_t *rcnt, *roff, *rcur;            // per body: neighbours in the entity graph, start of its list, fill cursor
    uint32_t *radj, *radj_m;                 // neighbour id | 0x80000000 if the adjacency holds a contact manifold; its manifold slot
    uint32_t *rstamp, *rnext;                // breadth-first walk: visit stamp and queue link per body

    // ---- narrowphase: manifold slots sorted by pair type (its own buffer: cidx_s, the solver order, outlives a step
    // whose island rebuild is skipped)
    uint32_t *npidx;

    // ---- materials: material::id per body (MATERIAL_UNASSIGNED = no id), and the material_mix_table as an open-addressing
    // hash of the unordered id pair (lo << 16 | hi) -> index into mix_mat (friction, restitution); mix_size slots
    uint32_t *matid;
    unsigned long long *mix_key; uint32_t *mix_idx; float2 *mix_mat; uint32_t mix_size;

    // ---- island-tile lane plan (k_tile_plan, part of the island rebuild).  Per tile: bodies, hinge lanes, contact
    // lanes, hinge colours | contact colours << 16.  Per tile lane (tile * TILE_CAP + t): the row header of hinge / manifold
    // t of the tile (tags, hinge id / manifold slot, record slots), and for each of the two its colour | the record slot
    // of its island's root << 16.
    uint4 *tile_hdr;
    uint4 *tplan_h, *tplan_c;
    uint2 *tplan_w;

    // ---- presentation transforms (present_position xyz, present_orientation xyzw) of the F_PRESENT bodies, written by
    // k_presentation between steps; appended last so that the step kernels' parameter offsets stay as they were
    float4 *ppos, *porn;
};

} // namespace b2d
